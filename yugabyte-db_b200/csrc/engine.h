// engine.h — host-side interface of the CUDA engine (implementation: engine.cu).
#pragma once
#include <mutex>
#include <string>
#include <vector>

#include "../../include/ybgpu_compaction.h"
#include "dev_logic.cuh"

namespace ybgpu {

constexpr int MAX_RUNS = 64;   // input files per job (configs use 2..32)
// opens the message of every failure caused by ybgpu_job_options::device_memory_budget (before upload or during run)
constexpr char kBudgetExceeded[] = "device memory budget exceeded";

// Device bytes held at once by a set of jobs (the ranges of one pipelined compaction): every allocation and free of a
// member job updates `in_use` when it happens, so `peak` is the high-water mark of the jobs' bytes live together.
struct MemGroup {
  std::mutex mu;
  uint64_t in_use = 0, peak = 0;
  void Change(int64_t delta) {
    std::lock_guard<std::mutex> l(mu);
    in_use += delta;
    if (in_use > peak) peak = in_use;
  }
};
// Makes `job` (a ybgpu_job of this library) a member of `group` from now until it is destroyed; its bytes held so far count.
void JoinMemGroup(ybgpu_job* job, MemGroup* group);

class Engine {
 public:
  explicit Engine(const ybgpu_job_options& o);
  ~Engine();
  ybgpu_status Init();
  ybgpu_status AddInput(const uint8_t* data, uint64_t len, const ybgpu_block_handle* handles, uint64_t nh,
                        int key_encoding, uint64_t ht_filter, bool on_device);
  ybgpu_status AddInputKv(const uint8_t* keys, const uint64_t* key_offsets, const uint8_t* values, const uint64_t* value_offsets, uint64_t n);
  void JoinMemGroup(MemGroup* group);
  ybgpu_status SetCotableFilters(const uint32_t* db_oids, const uint64_t* hybrid_times, uint32_t n);
  ybgpu_status WaitInputs();
  ybgpu_status Run(const volatile int32_t* shutting_down);
  ybgpu_status KvStreamSizes(uint64_t* n, uint64_t* kb, uint64_t* vb) const;
  ybgpu_status FetchKvStream(uint8_t* keys, uint64_t* koff, uint8_t* vals, uint64_t* voff);
  ybgpu_status Digest(uint64_t* digest);
  ybgpu_status OutputInfo(uint64_t* data_len, uint32_t* n_blocks, uint32_t* boundary_stride) const;
  ybgpu_status FetchOutput(uint8_t* data_file, uint64_t* block_off, uint8_t* boundary);
  // The finished data file, copied on a second stream so that the caller can build the metadata file
  // on the host while the DMA runs.
  ybgpu_status BeginFetchDataFile(uint8_t* data_file);
  ybgpu_status EndFetchDataFile();
  uint64_t kept_deletions() const;
  // smallest / largest internal key of the output as [u16 length][key] records (boundary stride of OutputInfo)
  ybgpu_status FetchFileBoundaries(uint8_t* smallest, uint8_t* largest);
  // Bloom filter blocks of the output (filter_policy != none): number of blocks, bytes per block
  // (bits + 5 metadata bytes), stride of the boundary key records.
  ybgpu_status FilterInfo(uint32_t* n_filter_blocks, uint32_t* block_bytes, uint32_t* key_stride) const;
  // filters: n*block_bytes; keys: per block [first key][last key] records ([u16 len][bytes], key_stride each);
  // first_entry[f]: output entry whose filter key opens block f; block_first[b]: first entry of data block b.
  ybgpu_status FetchFilter(uint8_t* filters, uint8_t* keys, uint32_t* first_entry, uint32_t* block_first);
  // FileMetaData user boundary values (options.compute_user_boundary_values): per range component, min / max value
  ybgpu_status FetchUserValues(ybgpu_user_value* smallest, ybgpu_user_value* largest, uint32_t cap, uint32_t* n);
  // Output check (verify_kernels.cuh): the finished table of this job, re-read in device memory and compared with the
  // merge result; and any split SST's data file from host memory (checksums, compressed streams, entries, key order).
  ybgpu_status VerifyOutput(ybgpu_output_check* result);
  ybgpu_status VerifySst(const uint8_t* data, uint64_t len, const ybgpu_block_handle* handles, uint64_t nh, int key_encoding,
                         ybgpu_output_check* result);
  const ybgpu_job_options& options() const { return opt_; }
  ybgpu_job_stats& stats();
  const std::string& error() const { return error_; }
  ybgpu_status Fail(ybgpu_status s, const std::string& msg);
  // a failed CUDA call (cudaError_t e); a request the job's device_memory_budget refused gets the budget message
  ybgpu_status FailCuda(const char* expr, int e);
  bool ran() const { return ran_; }
  int record_stride() const { return record_stride_; }
  uint32_t num_tiles() const { return num_tiles_; }

 private:
  ybgpu_status CheckDeviceError(const char* phase);
  ybgpu_status CheckBudgetBeforeUpload(uint64_t more);
  ybgpu_status ReadSmall(void* host_dst, const void* dev_src, size_t n);
  ybgpu_status UploadSmall(void* dev_dst, const void* host_src, size_t n);
  ybgpu_status ReadViaMapped(void* host_dst, const void* dev_src, size_t row_bytes, size_t src_pitch, size_t rows);
  ybgpu_status EnsureKvStream();
  ybgpu_status EnsureChunkSums();
  ybgpu_status VerifyTable(const uint8_t* file, uint64_t file_len, const unsigned long long* d_off, const uint32_t* d_size,
                           uint32_t nb, int key_encoding, bool job, ybgpu_output_check* result);
  struct Impl;
  ybgpu_job_options opt_;
  Impl* impl_;
  std::vector<uint8_t> largest_, lower_, upper_, range_lower_, range_upper_;
  ybgpu_job_stats stats_;
  std::string error_;
  bool ran_ = false;
  int record_stride_ = 0;
  uint32_t num_tiles_ = 0;
};

}  // namespace ybgpu
