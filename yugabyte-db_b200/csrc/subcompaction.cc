// subcompaction.cc — one compaction run as pipelined key-range subcompactions.
//
// Host-side replacement of CompactionJob::GenSubcompactionBoundaries and of the per-subcompaction
// threads of CompactionJob::Run (reference rocksdb/db/compaction_job.cc:409-519,532-552): the
// compaction is cut into key ranges on row boundaries, every range is an ordinary GPU job
// (ybgpu_job_*) over the data blocks of each input that can hold its keys, and the ranges run on a
// few host threads with a private CUDA stream each. While one range's inputs travel host->device,
// another range's kernels run and a third range's output travels device->host: PCIe is full duplex,
// so the end-to-end time of a large compaction approaches max(H2D, D2H) instead of their sum, and
// the device memory in use is bounded by `max_in_flight` ranges instead of the whole compaction.
// Everything here is host orchestration above the C ABI; no compaction logic runs on the CPU.
#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <chrono>
#include <cstdlib>
#include <cstdio>
#include <cstring>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/ybgpu_compaction.h"
#include "dev_logic.cuh"
#include "host_sst.h"
#include "engine.h"
#include "range_plan.h"

namespace ybgpu {
namespace plan {

using ybgpu::host::SstMeta;

std::string UserPart(const std::string& ikey) { return ikey.size() >= 8 ? ikey.substr(0, ikey.size() - 8) : ikey; }

bool ParseInputs(const ybgpu_input_file* files, uint32_t n, std::vector<ParsedInput>* out, std::string* err) {
  out->resize(n);
  std::vector<std::string> errs(n);
  auto parse_one = [&](uint32_t f) {
    ParsedInput& p = (*out)[f];
    std::string e = ybgpu::host::ParseSplitSstMeta(files[f].meta_file, files[f].meta_file_len, &p.meta);
    if (!e.empty()) { errs[f] = "input " + std::to_string(f) + ": " + e; return; }
    if (p.meta.separators.size() != p.meta.data_blocks.size()) { errs[f] = "index entries do not match data blocks"; return; }
    p.useps.reserve(p.meta.separators.size());
    for (const std::string& k : p.meta.separators) p.useps.push_back(UserPart(k));
    for (const auto& h : p.meta.data_blocks)
      if (h.offset > files[f].data_file_len || h.size > files[f].data_file_len - h.offset || files[f].data_file_len - h.offset - h.size < 5) {
        errs[f] = "block handle outside the data file"; return;
      }
  };
  // the index of a multi-GB input has ~10^5 entries: the files are walked side by side
  if (n > 1) {
    std::vector<std::thread> pool;
    for (uint32_t f = 0; f < n; f++) pool.emplace_back(parse_one, f);
    for (std::thread& t : pool) t.join();
  } else if (n == 1) {
    parse_one(0);
  }
  for (uint32_t f = 0; f < n; f++)
    if (!errs[f].empty()) { *err = errs[f]; return false; }
  return true;
}

// Weighted quantiles of the index separators, cut back to the row prefix. A splitter s must never
// fall inside a row (all entries of one DocKey D): that happens only if s = D + more bytes for the
// complete DocKey D of an existing row (a string between two strings that share the prefix D has
// the prefix D itself). The DocKey walk is a deterministic left-to-right parse, so
//   * if it succeeds on a separator, the separator is cut to that DocKey: a complete DocKey, of
//     which no other complete DocKey is a proper prefix;
//   * if it fails with a malformed key (FindShortestSeparator cut the separator inside a
//     component), the separator does not start with any complete DocKey and is used whole;
//   * if it stops at a key the engine does not take (vector-index metadata), the separator is skipped.
void CollectSamples(const std::vector<ParsedInput>& in, uint32_t n_ranges, std::vector<Sample>* samples) {
  // every stride-th separator of a file stands for the bytes of the blocks since the previous sample
  // (about 2^11 samples per range are plenty; a 30 GB compaction has ~10^6 index entries)
  size_t n_blocks = 0;
  for (const ParsedInput& p : in) n_blocks += p.useps.size();
  const size_t stride = std::max<size_t>(1, n_blocks / (static_cast<size_t>(std::max(1u, n_ranges)) << 11));
  for (const ParsedInput& p : in) {
    uint64_t w = 0;
    for (size_t i = 0; i < p.useps.size(); i++) {
      w += p.meta.data_blocks[i].size + 5;
      if ((i + 1) % stride == 0 || i + 1 == p.useps.size()) { samples->push_back({p.useps[i], w}); w = 0; }
    }
  }
}

bool RowPrefix(const std::string& k, bool docdb_keys, std::string* cut) {
  int plen = static_cast<int>(k.size());
  if (docdb_keys) {
    // group_prefix_len scans with aligned 8-byte loads: give it an aligned, padded copy
    alignas(8) uint8_t buf[1040];
    if (k.size() > 1024) return false;
    memset(buf, 0, sizeof(buf));
    memcpy(buf, k.data(), k.size());
    plen = ybgpu::group_prefix_len(buf, static_cast<int>(k.size()), true);
    if (plen == -ybgpu::DEV_ERR_UNSUPPORTED_KEY) return false;
    if (plen <= 0) plen = static_cast<int>(k.size());
  }
  if (plen == 0 || plen > YBGPU_MAX_SPLITTER_LEN) return false;
  *cut = k.substr(0, plen);
  return true;
}

std::vector<std::string> SplittersFromSamples(std::vector<Sample> samples, uint32_t n_ranges, bool docdb_keys) {
  std::vector<std::string> out;
  if (n_ranges <= 1 || samples.empty()) return out;
  uint64_t total = 0;
  for (const Sample& s : samples) total += s.w;
  std::sort(samples.begin(), samples.end(), [](const Sample& a, const Sample& b) { return a.key < b.key; });
  const double target = static_cast<double>(total) / n_ranges;
  double acc = 0, next = target;
  for (const Sample& s : samples) {
    acc += static_cast<double>(s.w);
    if (acc < next || out.size() + 1 >= n_ranges) continue;
    std::string cut;
    if (!RowPrefix(s.key, docdb_keys, &cut)) continue;
    if (!out.empty() && !(out.back() < cut)) continue;
    out.push_back(cut);
    next = target * static_cast<double>(out.size() + 1);
  }
  return out;
}

// The samples of the blocks that can hold keys of [lo, hi), already cut to their row prefix and kept only when that
// prefix lies strictly inside the range, then the weighted median of them.
bool SplitRange(const std::vector<ParsedInput>& in, const std::string& lo, const std::string& hi, bool docdb_keys, std::string* mid) {
  std::vector<Sample> samples;
  for (const ParsedInput& p : in) {
    size_t a, b;
    BlocksForRange(p.useps, lo, hi, &a, &b);
    uint64_t w = 0;
    for (size_t i = a; i < b; i++) {
      w += p.meta.data_blocks[i].size + 5;
      std::string cut;
      if (!RowPrefix(p.useps[i], docdb_keys, &cut) || !(lo < cut) || (!hi.empty() && !(cut < hi))) continue;
      samples.push_back({cut, w});
      w = 0;
    }
  }
  const std::vector<std::string> sp = SplittersFromSamples(std::move(samples), 2, false);
  if (sp.empty()) return false;
  *mid = sp[0];
  return true;
}

std::vector<std::string> PlanSplitters(const std::vector<ParsedInput>& in, uint32_t n_ranges, bool docdb_keys) {
  if (n_ranges <= 1) return {};
  std::vector<Sample> samples;
  CollectSamples(in, n_ranges, &samples);
  return SplittersFromSamples(std::move(samples), n_ranges, docdb_keys);
}

// Blocks [a, b) of one input that can hold user keys in [lo, hi): block i holds keys in
// (sep[i-1], sep[i]] (the separator is >= the block's last key and < the next block's first key).
void BlocksForRange(const std::vector<std::string>& useps, const std::string& lo, const std::string& hi, size_t* a, size_t* b) {
  const size_t nb = useps.size();
  *a = lo.empty() ? 0 : static_cast<size_t>(std::lower_bound(useps.begin(), useps.end(), lo) - useps.begin());
  if (hi.empty()) { *b = nb; return; }
  const size_t c = static_cast<size_t>(std::lower_bound(useps.begin(), useps.end(), hi) - useps.begin());
  *b = std::max(*a, std::min(nb, c + 1));
}

void SpansForRange(const ParsedInput& in, const std::string& lo, const std::string& hi, bool retention_enabled, std::vector<Span>* out) {
  out->clear();
  size_t a, b;
  BlocksForRange(in.useps, lo, hi, &a, &b);
  // A range that starts inside a cotable / colocated table ('y' + uuid or '0' + colocation id): the table's
  // tombstone entries `id ! # HT` sort before every row of the table, i.e. before this range, yet their
  // overwrite time (slot 0 of DocDBCompactionFeed's overwrite stack, docdb_compaction_context.cc:999-1024)
  // shadows the rows in it.
  if (retention_enabled && !lo.empty() && (lo[0] == 'y' || lo[0] == '0')) {
    const int id = ybgpu::dockey_id_size(reinterpret_cast<const uint8_t*>(lo.data()), static_cast<int>(lo.size()));
    if (id > 0 && static_cast<size_t>(id) <= lo.size()) {
      const std::string tomb_lo = lo.substr(0, id) + '!', tomb_hi = lo.substr(0, id) + '"';     // '!' + 1
      if (tomb_lo < lo) {                              // else the range starts at the tombstones themselves
        size_t ta, tb;
        BlocksForRange(in.useps, tomb_lo, tomb_hi, &ta, &tb);
        if (b <= a) { a = b = tb; }                    // no block of this file holds range keys
        tb = std::min(tb, a);
        if (tb > ta) {
          if (tb == a && b > a) a = ta;                // contiguous with the range's blocks: one span
          else out->push_back({ta, tb});
        }
      }
    }
  }
  if (b > a) out->push_back({a, b});
}

// Last internal key of one data block (BlockIter::SeekToLast: from the last restart point forward;
// table/block.cc:248-262,348-447 and block_internal.h:51-162 for three_shared_parts).
bool LastKeyOfBlock(const uint8_t* blk, uint64_t size, int key_encoding, std::string* key) {
  using namespace ybgpu;
  if (size < 8) return false;
  uint32_t num_restarts; memcpy(&num_restarts, blk + size - 4, 4);
  if (num_restarts == 0 || static_cast<uint64_t>(num_restarts) * 4 + 4 > size) return false;
  const uint32_t restarts_off = static_cast<uint32_t>(size - 4 - 4ull * num_restarts);
  uint32_t p; memcpy(&p, blk + restarts_off + 4ull * (num_restarts - 1), 4);
  if (p >= restarts_off) return false;
  std::string cur;
  bool first = true;
  while (p < restarts_off) {
    const uint32_t avail = restarts_off - p;
    if (key_encoding == YBGPU_KEY_ENCODING_THREE_SHARED_PARTS) {
      TspHeader th; uint32_t klen, ms, ml;
      const int h = parse_entry_header_tsp(blk + p, avail, &th);
      if (!h || (first && th.something_shared) || !tsp_key_layout(th, static_cast<uint32_t>(cur.size()), &klen, &ms, &ml)) return false;
      if (static_cast<uint64_t>(p) + h + th.ns1 + th.ns2 + th.vlen > restarts_off) return false;
      p += h;
      std::string nk;
      if (!th.something_shared) {
        nk.assign(reinterpret_cast<const char*>(blk + p), th.ns1);
      } else {
        uint64_t last = 0;
        if (th.last_size) {
          if (cur.size() < 8) return false;
          memcpy(&last, cur.data() + cur.size() - 8, 8);
          last += th.last_inc;
        }
        nk.assign(cur, 0, th.shared_prefix);
        nk.append(reinterpret_cast<const char*>(blk + p), th.ns1);
        nk.append(cur, ms, ml);
        nk.append(reinterpret_cast<const char*>(blk + p + th.ns1), th.ns2);
        if (th.last_size) nk.append(reinterpret_cast<const char*>(&last), 8);
      }
      if (nk.size() != klen) return false;
      cur.swap(nk);
      p += th.ns1 + th.ns2 + th.vlen;
    } else {
      uint32_t shared, non_shared, vlen;
      const int h = parse_entry_header(blk + p, avail, &shared, &non_shared, &vlen);
      if (!h || shared > cur.size() || (first && shared != 0)) return false;
      if (static_cast<uint64_t>(p) + h + non_shared + vlen > restarts_off) return false;
      p += h;
      cur.resize(shared);
      cur.append(reinterpret_cast<const char*>(blk + p), non_shared);
      p += non_shared + vlen;
    }
    first = false;
  }
  if (cur.size() < 8) return false;
  *key = cur;
  return true;
}

bool LastKeyOfFile(const ybgpu_input_file& f, const SstMeta& m, std::string* key, bool verify_checksum) {
  if (m.data_blocks.empty()) { key->clear(); return true; }
  const auto& h = m.data_blocks.back();
  if (h.offset > f.data_file_len || h.size > f.data_file_len - h.offset || f.data_file_len - h.offset - h.size < 5) return false;
  if (verify_checksum) {
    // ReadBlock verifies the stored bytes + type byte against the trailer before anything is decoded (table/format.cc:352-395;
    // ReadOptions::verify_checksums, which a compaction takes from verify_checksums_in_compaction)
    const uint8_t* p = f.data_file + h.offset;
    uint32_t stored;
    memcpy(&stored, p + h.size + 1, 4);
    if (ybgpu::host::Crc32cMask(ybgpu::host::Crc32c(p, h.size + 1)) != stored) return false;
  }
  const uint8_t type = f.data_file[h.offset + h.size];
  if (type != 0) {                                                  // stored compressed: uncompress on the host
    std::string raw;
    if (!ybgpu::host::UncompressStoredBlock(type, f.data_file + h.offset, h.size, &raw)) return false;
    return LastKeyOfBlock(reinterpret_cast<const uint8_t*>(raw.data()), raw.size(), m.key_encoding, key);
  }
  return LastKeyOfBlock(f.data_file + h.offset, h.size, m.key_encoding, key);
}

}  // namespace plan
}  // namespace ybgpu

namespace {

using namespace ybgpu::plan;
using ybgpu::host::SstMeta;

void AddStats(ybgpu_job_stats* t, const ybgpu_job_stats& s, bool first_output) {
  t->num_input_records += s.num_input_records; t->num_output_records += s.num_output_records;
  t->num_record_drop_hidden += s.num_record_drop_hidden; t->num_record_drop_obsolete += s.num_record_drop_obsolete;
  t->num_record_drop_feed += s.num_record_drop_feed;
  t->total_input_raw_key_bytes += s.total_input_raw_key_bytes; t->total_input_raw_value_bytes += s.total_input_raw_value_bytes;
  t->total_output_raw_key_bytes += s.total_output_raw_key_bytes; t->total_output_raw_value_bytes += s.total_output_raw_value_bytes;
  t->num_output_data_blocks += s.num_output_data_blocks;
  t->output_data_file_size += s.output_data_file_size; t->output_meta_file_size += s.output_meta_file_size;
  if (s.num_output_records) {
    t->smallest_seqno = first_output ? s.smallest_seqno : std::min(t->smallest_seqno, s.smallest_seqno);
    t->largest_seqno = std::max(t->largest_seqno, s.largest_seqno);
  }
  t->gpu_seconds += s.gpu_seconds; t->gpu_kernel_launches += s.gpu_kernel_launches;
  t->h2d_bytes += s.h2d_bytes; t->d2h_bytes += s.d2h_bytes;
  for (int i = 0; i < 8; i++) { t->phase_seconds[i] += s.phase_seconds[i]; t->phase_launches[i] += s.phase_launches[i]; }
  t->path_flags |= s.path_flags; t->tiles_inside_rows += s.tiles_inside_rows;
}

}  // namespace

extern "C" {

ybgpu_status ybgpu_sst_last_key(const uint8_t* meta_file, uint64_t meta_file_len, const uint8_t* data_file,
                                uint64_t data_file_len, uint8_t* key, uint32_t* key_len) {
  if (!meta_file || !data_file || !key || !key_len) return YBGPU_INVALID_ARGUMENT;
  SstMeta m;
  if (!ybgpu::host::ParseSplitSstMeta(meta_file, meta_file_len, &m).empty()) return YBGPU_CORRUPTION;
  ybgpu_input_file f{meta_file, meta_file_len, data_file, data_file_len, YBGPU_HT_INVALID, nullptr, nullptr, 0};
  std::string k;
  if (!LastKeyOfFile(f, m, &k) || k.size() > 1032) return YBGPU_CORRUPTION;
  memcpy(key, k.data(), k.size());
  *key_len = static_cast<uint32_t>(k.size());
  return YBGPU_OK;
}

ybgpu_status ybgpu_plan_subcompactions(const ybgpu_input_file* files, uint32_t num_files, uint32_t max_subcompactions,
                                       int32_t docdb_keys, uint8_t* splitters, uint32_t* splitter_lens,
                                       uint32_t* num_splitters) {
  if (!files || !splitters || !splitter_lens || !num_splitters) return YBGPU_INVALID_ARGUMENT;
  std::vector<ParsedInput> in;
  std::string err;
  if (!ParseInputs(files, num_files, &in, &err)) return YBGPU_CORRUPTION;
  const std::vector<std::string> sp = PlanSplitters(in, max_subcompactions, docdb_keys != 0);
  for (size_t i = 0; i < sp.size(); i++) {
    memcpy(splitters + 256 * i, sp[i].data(), sp[i].size());
    splitter_lens[i] = static_cast<uint32_t>(sp[i].size());
  }
  *num_splitters = static_cast<uint32_t>(sp.size());
  return YBGPU_OK;
}

ybgpu_status ybgpu_split_range(const ybgpu_input_file* files, uint32_t num_files, int32_t docdb_keys, const uint8_t* lower,
                               uint32_t lower_len, const uint8_t* upper, uint32_t upper_len, uint8_t* splitter, uint32_t* splitter_len) {
  if (!files || !splitter || !splitter_len || (lower_len && !lower) || (upper_len && !upper)) return YBGPU_INVALID_ARGUMENT;
  std::vector<ParsedInput> in;
  std::string err;
  if (!ParseInputs(files, num_files, &in, &err)) return YBGPU_CORRUPTION;
  std::string mid;
  const std::string lo(reinterpret_cast<const char*>(lower), lower_len), hi(reinterpret_cast<const char*>(upper), upper_len);
  if (!SplitRange(in, lo, hi, docdb_keys != 0, &mid)) return YBGPU_NOT_FOUND;
  memcpy(splitter, mid.data(), mid.size());
  *splitter_len = static_cast<uint32_t>(mid.size());
  return YBGPU_OK;
}

}  // extern "C"

namespace {

// ONE output table: the range data files land back to back in the caller's buffer (a range's D2H target is known as
// soon as every earlier range knows its size) and a ConcatBuilder consumes the ranges in key order as they complete.
struct OneTable {
  std::string meta;                     // result: the one metadata file
  uint64_t data_len = 0;
  uint32_t pieces = 0;
  std::string smallest, largest;
};

ybgpu_status CompactFilesCore(const ybgpu_job_options* options, const ybgpu_input_file* files, uint32_t num_files,
                              uint32_t max_subcompactions, uint32_t max_in_flight,
                              uint8_t* data_arena, uint64_t data_arena_cap, uint8_t* meta_arena, uint64_t meta_arena_cap,
                              const volatile int32_t* shutting_down, ybgpu_sub_output* outputs, uint32_t* num_outputs,
                              ybgpu_job_stats* total, char* err, uint64_t err_cap, OneTable* one, bool verify_outputs) {
  auto fail = [&](ybgpu_status s, const std::string& msg) {
    if (err && err_cap) snprintf(err, err_cap, "%s", msg.c_str());
    return s;
  };
  if (!options || !files || !outputs || !num_outputs || !data_arena || (!meta_arena && !one)) return fail(YBGPU_INVALID_ARGUMENT, "null argument");
  if (options->range_lower_len || options->range_upper_len) return fail(YBGPU_INVALID_ARGUMENT, "range bounds are set by the subcompaction planner");
  if (!ybgpu::host::OutputCompressionSupported(options->output_compression))
    return fail(YBGPU_NOT_SUPPORTED, ybgpu::host::UnsupportedOutputCompression(options->output_compression));
  const uint64_t budget = options->device_memory_budget;
  if (max_subcompactions == 0 && !budget) max_subcompactions = 1;
  const uint32_t output_slots = budget && !one ? *num_outputs : max_subcompactions;
  if (max_in_flight == 0) max_in_flight = 3;
  // every range runs as a job with this budget (its reservation until it has run)
  const uint64_t job_budget = budget ? std::max<uint64_t>(1, budget / max_in_flight) : 0;
  std::vector<ParsedInput> in;
  std::string perr;
  if (!ParseInputs(files, num_files, &in, &perr)) return fail(YBGPU_CORRUPTION, perr);
  if (max_subcompactions == 0) {
    // as many ranges as the budget needs: about a third of a range's budget in input bytes (inputs + uncompressed image);
    // a range that needs more is cut again when it runs
    uint64_t known = 0;
    for (uint32_t f = 0; f < num_files; f++) {
      uint64_t comp = 0;
      const uint64_t img = ybgpu::host::UncompressedImageBytes(files[f].data_file, in[f].meta.data_blocks.data(), in[f].meta.data_blocks.size(), &comp);
      known += files[f].data_file_len + (comp ? img : 0);
    }
    const uint64_t per_range = std::max<uint64_t>(1, job_budget / 3);
    max_subcompactions = static_cast<uint32_t>(std::min<uint64_t>(1u << 16, std::max<uint64_t>(1, (known + per_range - 1) / per_range)));
  }

  // Compaction::GetLargestUserKey (db/compaction.cc:318): the seqno-zeroing exception key is a
  // property of the whole compaction, not of a range.
  std::string largest_user;
  bool have_largest = options->has_largest_user_key != 0;
  if (have_largest) {
    largest_user.assign(reinterpret_cast<const char*>(options->largest_user_key), options->largest_user_key_len);
  } else {
    for (uint32_t f = 0; f < num_files; f++) {
      std::string k;
      if (!LastKeyOfFile(files[f], in[f].meta, &k, options->verify_checksums != 0)) return fail(YBGPU_CORRUPTION, "cannot read the last key of input " + std::to_string(f));
      if (k.empty()) continue;
      std::string u = UserPart(k);
      if (!have_largest || largest_user < u) { largest_user = u; have_largest = true; }
    }
  }

  const bool docdb_keys = options->retention_enabled != 0;
  const std::vector<std::string> splitters = PlanSplitters(in, max_subcompactions, docdb_keys);
  const uint32_t n_ranges = static_cast<uint32_t>(splitters.size()) + 1;
  if (n_ranges > output_slots && !one) return fail(YBGPU_INVALID_ARGUMENT, "more ranges than output slots");
  *num_outputs = n_ranges;
  // the outputs of every planned range in key order: one, or more when the range was cut to fit the budget
  std::vector<std::vector<ybgpu_sub_output>> subs(n_ranges);

  // device_memory_budget: ranges are admitted in range order while the reservations on the device leave room; a range
  // holds job_budget until it has run, then its measured peak until its job is destroyed
  std::mutex res_mu;
  std::condition_variable res_cv;
  uint64_t reserved = 0;
  auto reserve = [&](uint64_t x) {
    std::unique_lock<std::mutex> l(res_mu);
    res_cv.wait(l, [&] { return reserved + x <= budget; });
    reserved += x;
  };
  auto unreserve = [&](uint64_t x) {
    { std::lock_guard<std::mutex> l(res_mu); reserved -= x; }
    res_cv.notify_all();
  };
  // every range job counts its allocations and frees here as well: total.device_bytes_peak is the high-water mark of the
  // bytes the ranges hold at once
  ybgpu::MemGroup mem_group;

  std::atomic<uint32_t> next_range{0};
  std::atomic<uint64_t> data_used{0}, meta_used{0};
  std::atomic<bool> failed{false};
  std::mutex err_mu;
  ybgpu_status first_status = YBGPU_OK;
  std::string first_error;
  // one-table mode: per-range progress (0 running, 1 output size known, 2 complete) and the assembler
  std::mutex ot_mu;
  std::condition_variable ot_cv;
  std::vector<int> ot_state(one ? n_ranges : 0, 0);
  std::vector<uint64_t> ot_dlen(one ? n_ranges : 0, 0);             // the range's data bytes, all its pieces
  std::vector<std::vector<std::string>> ot_meta(one ? n_ranges : 0); // per piece of the range
  uint32_t ot_next = 0;
  size_t ot_next_piece = 0;
  std::unique_ptr<ybgpu::host::ConcatBuilder> ot_builder;
  std::string ot_error;
  auto record_failure = [&](ybgpu_status s, const std::string& msg) {
    {
      std::lock_guard<std::mutex> lock(err_mu);
      if (!failed.exchange(true)) { first_status = s; first_error = msg; }
    }
    if (one) { std::lock_guard<std::mutex> lock(ot_mu); ot_cv.notify_all(); }
  };
  ybgpu::host::TableOptions ot_topt;
  if (one) {
    ot_topt.block_size = options->block_size; ot_topt.block_restart_interval = options->block_restart_interval;
    ot_topt.block_size_deviation = options->block_size_deviation; ot_topt.index_block_size = options->index_block_size;
    ot_topt.min_keys_per_index_block = options->min_keys_per_index_block; ot_topt.key_encoding = options->output_key_encoding;
    ot_topt.filter_policy = options->filter_policy; if (options->filter_block_size) ot_topt.filter_block_size = options->filter_block_size; ot_topt.compression = options->output_compression;
    ot_builder.reset(new ybgpu::host::ConcatBuilder(ot_topt));
    uint64_t in_meta = 0;
    for (uint32_t f = 0; f < num_files; f++) in_meta += files[f].meta_file_len;
    ot_builder->Reserve(in_meta + in_meta / 4 + 65536);
  }
  auto ot_piece = [&](uint32_t r, size_t i) {
    const ybgpu_sub_output& o = subs[r][i];
    ybgpu::host::SstPiece p;
    p.meta = reinterpret_cast<const uint8_t*>(ot_meta[r][i].data()); p.meta_len = ot_meta[r][i].size(); p.data_len = o.data_len;
    p.smallest.assign(reinterpret_cast<const char*>(o.smallest_key), o.smallest_key_len);
    p.largest.assign(reinterpret_cast<const char*>(o.largest_key), o.largest_key_len);
    return p;
  };
  // With ot_mu held: the first piece with data at or after piece i of range a -> (*ra, *ri); false when a range on the way
  // has not completed. (*ra == n_ranges: none is left.)
  auto ot_seek = [&](uint32_t a, size_t i, uint32_t* ra, size_t* ri) {
    for (; a < n_ranges; a++, i = 0) {
      *ra = a; *ri = i;
      if (ot_state[a] != 2) return false;
      for (; i < subs[a].size(); i++)
        if (subs[a][i].data_len) { *ri = i; return true; }
    }
    *ra = n_ranges; *ri = 0;
    return true;
  };
  // Called with ot_mu held (through `lock`): feeds every piece whose successor is known to the builder, in key order.
  // The assembly itself (index keys rebased, separators recomputed: milliseconds per piece) runs WITHOUT ot_mu — the
  // other ranges publish their sizes and learn their offsets under that mutex — by whichever thread finds no assembler
  // active; that thread keeps going until no further piece is ready.
  bool ot_building = false;
  auto ot_advance = [&](std::unique_lock<std::mutex>& lock) {
    if (ot_building) return;
    ot_building = true;
    while (ot_error.empty()) {
      uint32_t a, nx;
      size_t i, ni;
      if (!ot_seek(ot_next, ot_next_piece, &a, &i)) break;
      if (a >= n_ranges) { ot_next = n_ranges; break; }
      if (!ot_seek(a, i + 1, &nx, &ni)) break;                      // the successor's first key is not known yet
      const ybgpu::host::SstPiece pa = ot_piece(a, i);
      ybgpu::host::SstPiece pn;
      if (nx < n_ranges) pn = ot_piece(nx, ni);
      lock.unlock();
      std::string e = ot_builder->AddPiece(pa, nx < n_ranges ? &pn : nullptr);
      lock.lock();
      ot_error = e;
      if (one->pieces == 0) one->smallest = pa.smallest;
      one->largest = pa.largest;
      one->pieces++;
      std::string().swap(ot_meta[a][i]);                            // the piece's own metadata file is no longer needed
      ot_next = nx; ot_next_piece = ni;
    }
    ot_building = false;
  };

  const bool trace = getenv("YBGPU_SUB_TRACE") != nullptr;      // per-range timeline on stderr (ms since the call)
  const auto t_start = std::chrono::steady_clock::now();
  auto ms_now = [&]() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_start).count(); };
  if (trace) fprintf(stderr, "[ybgpu sub] planned %u ranges at %.1f ms\n", n_ranges, ms_now());

  // Copy slots. A copy engine serves the streams that have copies pending chunk by chunk in turn: with every range in
  // flight queueing its inputs at once, all of them receive their data at the same (late) time, compute together and
  // copy out together — the pipeline moves in convoys and each direction idles while the other ramps. Instead at most
  // `h2d_slots` ranges have inputs in transit (taken in range order; default 1: a range's inputs arrive at the full
  // link rate) and at most `d2h_slots` copy out (default 2), so the first range computes after ONE range's worth of DMA
  // and both directions stay busy from then on (profiles/r02_e2e_sweep_100m*.jsonl).
  struct Slots {
    std::mutex mu; std::condition_variable cv; uint32_t free_slots;
    explicit Slots(uint32_t n) : free_slots(n) {}
    void Acquire() { std::unique_lock<std::mutex> l(mu); cv.wait(l, [&] { return free_slots > 0; }); free_slots--; }
    void Release() { { std::lock_guard<std::mutex> l(mu); free_slots++; } cv.notify_one(); }
  };
  struct SlotGuard {
    Slots* s = nullptr;
    void Take(Slots* x) { x->Acquire(); s = x; }
    void Drop() { if (s) { s->Release(); s = nullptr; } }
    ~SlotGuard() { Drop(); }
  };
  auto env_u32 = [](const char* name, uint32_t dflt) {
    const char* v = getenv(name);
    if (!v || !*v) return dflt;
    const long x = atol(v);
    return x <= 0 ? 0u : static_cast<uint32_t>(x);
  };
  const uint32_t h2d_slots = env_u32("YBGPU_H2D_SLOTS", 1), d2h_slots = env_u32("YBGPU_D2H_SLOTS", 2);   // 0 = ungated
  Slots h2d_gate(h2d_slots ? h2d_slots : 1u << 30), d2h_gate(d2h_slots ? d2h_slots : 1u << 30);
  // ranges take their input slot in range order (a later range must not overtake: its output offset waits on the
  // earlier ones in one-table mode)
  std::mutex order_mu; std::condition_variable order_cv; uint32_t h2d_next = 0;

  auto run_range = [&](uint32_t r) {
    // input slot (and, under a budget, the range's reservation), in range order; every range that was handed out passes
    // here, so nobody waits for a range that gave up
    SlotGuard in_slot, out_slot;
    {
      std::unique_lock<std::mutex> lock(order_mu);
      order_cv.wait(lock, [&] { return h2d_next == r; });
    }
    uint64_t held = 0;                                        // this range's reservation
    if (budget) { reserve(job_budget); held = job_budget; }
    in_slot.Take(&h2d_gate);
    {
      std::lock_guard<std::mutex> lock(order_mu);
      h2d_next = r + 1;
    }
    order_cv.notify_all();
    struct Unreserve { std::function<void()> f; ~Unreserve() { f(); } } unreserve_at_exit{[&] { if (held) unreserve(held); }};
    // the key ranges still to run for this planned range, the next one at the back: one, unless a job needs more than
    // its budget and the range is cut in two
    std::vector<std::pair<std::string, std::string>> todo;
    todo.emplace_back(r > 0 ? splitters[r - 1] : std::string(), r + 1 < n_ranges ? splitters[r] : std::string());
    uint64_t r_data = 0;                                      // one-table mode: data bytes of this range's earlier pieces
    bool first_piece = true;
    while (!todo.empty()) {
      const std::string lo = todo.back().first, hi = todo.back().second;
      todo.pop_back();
      if (!first_piece) in_slot.Take(&h2d_gate);
      first_piece = false;
      ybgpu_sub_output out;
      memset(&out, 0, sizeof(out));
      out.range_lower_len = static_cast<uint32_t>(lo.size()); memcpy(out.range_lower, lo.data(), lo.size());
      out.range_upper_len = static_cast<uint32_t>(hi.size()); memcpy(out.range_upper, hi.data(), hi.size());
      double t_begin = ms_now(), t_added = 0, t_ran = 0, t_sized = 0, t_d2h = 0, t_fetched = 0;
      ybgpu_job_options o = *options;
      o.cuda_stream = YBGPU_STREAM_PRIVATE;
      o.range_lower = out.range_lower; o.range_lower_len = out.range_lower_len;
      o.range_upper = out.range_upper; o.range_upper_len = out.range_upper_len;
      o.has_largest_user_key = have_largest ? 1 : 0;
      o.largest_user_key = reinterpret_cast<const uint8_t*>(largest_user.data());
      o.largest_user_key_len = largest_user.size();
      o.device_memory_budget = job_budget;
      ybgpu_job* job = nullptr;
      ybgpu_status s = ybgpu_job_create(&o, &job);
      if (s != YBGPU_OK) { record_failure(s, std::string("create: ") + ybgpu_last_error()); return; }
      ybgpu::JoinMemGroup(job, &mem_group);
      auto destroy = [&]() { ybgpu_job_destroy(job); };
      // true: the range was cut in two and both halves wait in `todo` (the job needed more than its budget)
      bool cut = false;
      // may_cut: the calls that allocate device memory (add_input, run, verify_output); a budget failure anywhere else
      // fails the compaction like any other error
      auto job_fail = [&](ybgpu_status st, const char* what, bool may_cut = false) {
        const std::string msg = ybgpu_job_error(job);
        destroy();
        if (may_cut && budget && msg.find(ybgpu::kBudgetExceeded) != std::string::npos) {
          std::string mid;
          if (SplitRange(in, lo, hi, docdb_keys, &mid)) {
            todo.emplace_back(mid, hi);
            todo.emplace_back(lo, mid);
            cut = true;
            return;
          }
          record_failure(st, std::string(what) + " (range " + std::to_string(r) + ", no row boundary left to cut it at): " + msg);
          return;
        }
        record_failure(st, std::string(what) + " (range " + std::to_string(r) + "): " + msg);
      };
      auto failed_or_cut = [&]() { in_slot.Drop(); return !cut; };
      uint32_t added = 0;
      std::vector<ybgpu_block_handle> h;

      // the blocks of every input that can hold keys of the range, plus — for a range that starts inside a cotable —
      // the blocks with that table's tombstones (SpansForRange); the last span of an input is its range span
      std::vector<Span> spans;
      for (uint32_t f = 0; f < num_files; f++) {
        SpansForRange(in[f], lo, hi, options->retention_enabled != 0, &spans);
        const auto& blocks = in[f].meta.data_blocks;
        for (const Span& sp : spans) {
          const uint64_t start = blocks[sp.a].offset;
          const uint64_t end = blocks[sp.b - 1].offset + blocks[sp.b - 1].size + 5;
          h.resize(sp.b - sp.a);
          for (size_t i = sp.a; i < sp.b; i++) { h[i - sp.a].offset = blocks[i].offset - start; h[i - sp.a].size = blocks[i].size; }
          s = ybgpu_job_add_input(job, files[f].data_file + start, end - start, h.data(), h.size(), in[f].meta.key_encoding, files[f].hybrid_time_filter);
          if (s != YBGPU_OK) { job_fail(s, "add_input", true); if (failed_or_cut()) return; break; }
          if (files[f].num_cotable_filters) {
            s = ybgpu_job_set_cotable_filters(job, files[f].cotable_db_oids, files[f].cotable_hybrid_times, static_cast<uint32_t>(files[f].num_cotable_filters));
            if (s != YBGPU_OK) { job_fail(s, "set_cotable_filters"); return; }
          }
          added++;
        }
        if (cut) break;
      }
      if (cut) continue;
      if (added && h2d_slots) {
        s = ybgpu_job_wait_inputs(job);
        if (s != YBGPU_OK) { job_fail(s, "wait_inputs"); return; }
      }
      in_slot.Drop();
      t_added = ms_now();
      if (added) {
        s = ybgpu_job_run(job, shutting_down);
        if (s != YBGPU_OK) { job_fail(s, "run", true); if (failed_or_cut()) return; continue; }
        if (verify_outputs) {
          // paranoid_file_checks: the range's table is re-read on its own stream while it is still in device memory; a bad
          // range fails the compaction before a byte of it reaches the caller's arena
          ybgpu_output_check chk;
          s = ybgpu_job_verify_output(job, &chk);
          if (s != YBGPU_OK) { job_fail(s, "verify_output", true); if (failed_or_cut()) return; continue; }
        }
        if (held && todo.empty()) {
          // the range has run: from here on it holds no more than what it measured
          ybgpu_job_stats st;
          ybgpu_job_get_stats(job, &st);
          const uint64_t peak = std::min(held, st.device_bytes_peak);
          unreserve(held - peak);
          held = peak;
        }
        t_ran = ms_now();
        uint64_t dl = 0, ml = 0;
        s = ybgpu_job_output_sizes(job, &dl, &ml);
        if (s != YBGPU_OK) { job_fail(s, "output_sizes"); return; }
        t_sized = ms_now();
        uint64_t doff = 0, moff = 0;
        uint8_t* meta_dst = nullptr;
        std::string piece_meta;
        if (one) {
          // this range's bytes follow those of every earlier range: wait until they all know their sizes (and publish this
          // range's once its last piece is sized)
          std::unique_lock<std::mutex> lock(ot_mu);
          if (todo.empty()) { ot_dlen[r] = r_data + dl; ot_state[r] = 1; ot_cv.notify_all(); }
          ot_cv.wait(lock, [&] {
            if (failed.load()) return true;
            for (uint32_t q = 0; q < r; q++) if (ot_state[q] == 0) return false;
            return true;
          });
          if (failed.load()) { lock.unlock(); destroy(); return; }
          for (uint32_t q = 0; q < r; q++) doff += ot_dlen[q];
          doff += r_data;
          r_data += dl;
          piece_meta.resize(ml);
          meta_dst = reinterpret_cast<uint8_t*>(&piece_meta[0]);
        }
        if (dl) {
          if (!one) {
            // 4 KB aligned slices of the caller's arenas, handed out in completion order
            doff = data_used.fetch_add((dl + 4095) & ~4095ull);
            moff = meta_used.fetch_add((ml + 4095) & ~4095ull);
            if (moff + ml > meta_arena_cap) { job_fail(YBGPU_INVALID_ARGUMENT, "output arena too small"); return; }
            meta_dst = meta_arena + moff;
          }
          if (doff + dl > data_arena_cap) { job_fail(YBGPU_INVALID_ARGUMENT, "output arena too small"); return; }
          out_slot.Take(&d2h_gate);
          t_d2h = ms_now();
          s = ybgpu_job_fetch_output(job, data_arena + doff, dl, meta_dst, ml);
          out_slot.Drop();
          if (s != YBGPU_OK) { job_fail(s, "fetch_output"); return; }
          out.data_offset = doff; out.data_len = dl; out.meta_offset = moff; out.meta_len = ml;
          uint64_t sl = 0, ll = 0;
          uint8_t sk[4096], lk[4096];
          s = ybgpu_job_output_boundaries(job, sk, &sl, lk, &ll);
          if (s != YBGPU_OK) { job_fail(s, "output_boundaries"); return; }
          out.smallest_key_len = static_cast<uint32_t>(std::min<uint64_t>(sl, sizeof(out.smallest_key)));
          out.largest_key_len = static_cast<uint32_t>(std::min<uint64_t>(ll, sizeof(out.largest_key)));
          memcpy(out.smallest_key, sk, out.smallest_key_len);
          memcpy(out.largest_key, lk, out.largest_key_len);
        }
        t_fetched = ms_now();
        ybgpu_job_get_stats(job, &out.stats);
        if (one) ot_meta[r].push_back(std::move(piece_meta));
      } else if (one) {
        std::lock_guard<std::mutex> lock(ot_mu);
        if (todo.empty()) { ot_dlen[r] = r_data; ot_state[r] = 1; ot_cv.notify_all(); }
        ot_meta[r].emplace_back();
      }
      destroy();
      subs[r].push_back(out);
      const double t_destroyed = ms_now();
      if (trace)
        fprintf(stderr, "[ybgpu sub] range %2u.%zu: begin %7.1f  inputs in %7.1f  run done %7.1f  meta built %7.1f  d2h start %7.1f  output fetched %7.1f  destroyed %7.1f  (gpu %.1f ms, %.2f GB in)\n",
                r, subs[r].size() - 1, t_begin, t_added, t_ran, t_sized, t_d2h, t_fetched, t_destroyed, out.stats.gpu_seconds * 1e3, out.stats.h2d_bytes / 1e9);
    }
    if (held) { unreserve(held); held = 0; }
    if (one) {
      std::unique_lock<std::mutex> lock(ot_mu);
      ot_state[r] = 2;
      ot_cv.notify_all();
      ot_advance(lock);
    }
  };

  auto worker = [&](bool pool_thread) {
    if (pool_thread) ybgpu_bind_thread_to_device(options->device, nullptr, nullptr);   // never the caller's own thread
    for (;;) {
      if (failed.load()) return;
      if (options->yield_fn) options->yield_fn(options->yield_ctx);      // PauseIfNecessary between ranges
      if (shutting_down && *shutting_down) { record_failure(YBGPU_SHUTDOWN_IN_PROGRESS, "Database shutdown or Column family drop during compaction"); return; }
      const uint32_t r = next_range.fetch_add(1);
      if (r >= n_ranges) return;
      run_range(r);
    }
  };
  const uint32_t n_threads = std::min(max_in_flight, n_ranges);
  if (n_threads <= 1) {
    worker(false);
  } else {
    std::vector<std::thread> pool;
    for (uint32_t t = 0; t < n_threads; t++) pool.emplace_back(worker, true);
    for (std::thread& t : pool) t.join();
  }
  if (failed.load()) return fail(first_status, first_error);
  if (one) {
    std::unique_lock<std::mutex> lock(ot_mu);
    ot_advance(lock);
    if (!ot_error.empty()) return fail(YBGPU_INVALID_ARGUMENT, "one-table assembly: " + ot_error);
    if (ot_next != n_ranges) return fail(YBGPU_RUNTIME_ERROR, "one-table assembly did not consume every range");
    for (uint32_t r = 0; r < n_ranges; r++) one->data_len += ot_dlen[r];
    if (one->pieces) {
      const std::string e = ot_builder->Finish(&one->meta);
      if (!e.empty()) return fail(YBGPU_INVALID_ARGUMENT, "one-table assembly: " + e);
    }
  }
  uint32_t n_out = 0;
  for (uint32_t r = 0; r < n_ranges; r++) n_out += static_cast<uint32_t>(subs[r].size());
  if (!one) {
    if (n_out > output_slots) return fail(YBGPU_INVALID_ARGUMENT, "the budget needed " + std::to_string(n_out) + " ranges, outputs has " +
                                                                      std::to_string(output_slots) + " slots");
    uint32_t i = 0;
    for (uint32_t r = 0; r < n_ranges; r++)
      for (const ybgpu_sub_output& o : subs[r]) outputs[i++] = o;
  }
  *num_outputs = n_out;
  if (total) {
    memset(total, 0, sizeof(*total));
    bool first_output = true;
    for (uint32_t r = 0; r < n_ranges; r++)
      for (const ybgpu_sub_output& o : subs[r]) {
        AddStats(total, o.stats, first_output);
        if (o.stats.num_output_records) first_output = false;
      }
    total->device_bytes_peak = mem_group.peak;
  }
  return YBGPU_OK;
}

}  // namespace

extern "C" {

ybgpu_status ybgpu_compact_files(const ybgpu_job_options* options, const ybgpu_input_file* files, uint32_t num_files,
                                 uint32_t max_subcompactions, uint32_t max_in_flight,
                                 uint8_t* data_arena, uint64_t data_arena_cap, uint8_t* meta_arena, uint64_t meta_arena_cap,
                                 const volatile int32_t* shutting_down, ybgpu_sub_output* outputs, uint32_t* num_outputs,
                                 ybgpu_job_stats* total, char* err, uint64_t err_cap) {
  return CompactFilesCore(options, files, num_files, max_subcompactions, max_in_flight, data_arena, data_arena_cap, meta_arena,
                          meta_arena_cap, shutting_down, outputs, num_outputs, total, err, err_cap, nullptr, false);
}

static ybgpu_status CompactFilesOneTable(const ybgpu_job_options* options, const ybgpu_input_file* files, uint32_t num_files,
                                           uint32_t max_subcompactions, uint32_t max_in_flight,
                                           uint8_t* data_out, uint64_t data_cap, uint8_t* meta_out, uint64_t meta_cap,
                                           const volatile int32_t* shutting_down, ybgpu_one_table_result* result,
                                           ybgpu_job_stats* total, char* err, uint64_t err_cap, bool verify_outputs) {
  if (!result || !data_out || !meta_out) { if (err && err_cap) snprintf(err, err_cap, "null argument"); return YBGPU_INVALID_ARGUMENT; }
  memset(result, 0, sizeof(*result));
  std::vector<ybgpu_sub_output> outs(1);                 // unused: one-table mode keeps the range outputs to itself
  uint32_t n = 0;
  OneTable one;
  ybgpu_job_stats tot;
  ybgpu_status s = CompactFilesCore(options, files, num_files, max_subcompactions, max_in_flight, data_out, data_cap, nullptr, 0,
                                    shutting_down, outs.data(), &n, &tot, err, err_cap, &one, verify_outputs);
  if (s != YBGPU_OK) return s;
  if (one.meta.size() > meta_cap) { if (err && err_cap) snprintf(err, err_cap, "metadata buffer too small"); return YBGPU_INVALID_ARGUMENT; }
  memcpy(meta_out, one.meta.data(), one.meta.size());
  result->data_len = one.data_len; result->meta_len = one.meta.size();
  result->num_ranges = n; result->num_pieces = one.pieces;
  result->smallest_key_len = static_cast<uint32_t>(std::min<size_t>(one.smallest.size(), sizeof(result->smallest_key)));
  result->largest_key_len = static_cast<uint32_t>(std::min<size_t>(one.largest.size(), sizeof(result->largest_key)));
  memcpy(result->smallest_key, one.smallest.data(), result->smallest_key_len);
  memcpy(result->largest_key, one.largest.data(), result->largest_key_len);
  tot.output_data_file_size = one.data_len; tot.output_meta_file_size = one.meta.size();
  if (total) *total = tot;
  return YBGPU_OK;
}

ybgpu_status ybgpu_compact_files_one_table(const ybgpu_job_options* options, const ybgpu_input_file* files, uint32_t num_files,
                                           uint32_t max_subcompactions, uint32_t max_in_flight,
                                           uint8_t* data_out, uint64_t data_cap, uint8_t* meta_out, uint64_t meta_cap,
                                           const volatile int32_t* shutting_down, ybgpu_one_table_result* result,
                                           ybgpu_job_stats* total, char* err, uint64_t err_cap) {
  return CompactFilesOneTable(options, files, num_files, max_subcompactions, max_in_flight, data_out, data_cap, meta_out, meta_cap, shutting_down,
                              result, total, err, err_cap, false);
}

ybgpu_status ybgpu_compact_files_checked(const ybgpu_job_options* options, const ybgpu_input_file* files, uint32_t num_files,
                                         uint32_t max_subcompactions, uint32_t max_in_flight,
                                         uint8_t* data_arena, uint64_t data_arena_cap, uint8_t* meta_arena, uint64_t meta_arena_cap,
                                         const volatile int32_t* shutting_down, ybgpu_sub_output* outputs, uint32_t* num_outputs,
                                         ybgpu_job_stats* total, char* err, uint64_t err_cap, int32_t verify_outputs) {
  return CompactFilesCore(options, files, num_files, max_subcompactions, max_in_flight, data_arena, data_arena_cap, meta_arena,
                          meta_arena_cap, shutting_down, outputs, num_outputs, total, err, err_cap, nullptr, verify_outputs != 0);
}

ybgpu_status ybgpu_compact_files_one_table_checked(const ybgpu_job_options* options, const ybgpu_input_file* files, uint32_t num_files,
                                                   uint32_t max_subcompactions, uint32_t max_in_flight,
                                                   uint8_t* data_out, uint64_t data_cap, uint8_t* meta_out, uint64_t meta_cap,
                                                   const volatile int32_t* shutting_down, ybgpu_one_table_result* result,
                                                   ybgpu_job_stats* total, char* err, uint64_t err_cap, int32_t verify_outputs) {
  return CompactFilesOneTable(options, files, num_files, max_subcompactions, max_in_flight, data_out, data_cap, meta_out, meta_cap, shutting_down,
                              result, total, err, err_cap, verify_outputs != 0);
}

}  // extern "C"
