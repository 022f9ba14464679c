// range_exchange.cc — one oversized compaction, key-range sharded across the GPUs of a box (SURVEY.md 8e,
// BASELINE config 5): "a single oversized tablet's major compaction is key-range-sharded across GPUs with one NCCL
// alltoall over NVLink to exchange boundary runs".
//
// Every rank starts with some of the tablet's input files in its host memory (files are staged round-robin).
//   1. plan      each rank samples the index separators of its files (range_plan.h: CollectSamples), the samples are
//                all-gathered through the communicator and every rank derives the SAME world x rounds - 1 row-aligned
//                splitters (SplittersFromSamples — the GPU analogue of CompactionJob::GenSubcompactionBoundaries,
//                rocksdb/db/compaction_job.cc:409-519). Rank d owns the `rounds` consecutive key ranges
//                [d * rounds, (d + 1) * rounds): the ranks' outputs are in key order, like the sub-outputs the
//                reference installs in order (compaction_job.cc:1128-1131).
//   2. exchange  per round t, for every (local file, destination rank): the contiguous run of data blocks that can
//                hold keys of the destination's range t (plus the table tombstone blocks of a range that starts
//                inside a cotable) travels ONCE: host -> device staging in chunks -> grouped ncclSend / ncclRecv over
//                NVLink -> the destination's HBM. Counts first (one all-gather of the byte matrix), then the block
//                handles, then the data, chunked so that staging memory is bounded.
//   3. compact   the destination runs an ordinary job over the slices it received (add_input_device) with
//                range_lower / range_upper set: entries of boundary blocks outside the range are invisible.
//   4. assemble  a rank's `rounds` outputs are concatenated into ONE table per rank (ConcatBuilder): with rounds > 1 a
//                rank never holds more than 1 / (world * rounds) of the compaction in HBM — that is how an input
//                larger than the GPUs' memory (1 TB over 8 x 180 GB) goes through.
// The seqno-zeroing exception key (Compaction::GetLargestUserKey, db/compaction.cc:318) is the maximum over all ranks.
//
// NCCL is loaded at run time (dlopen) so that single-GPU users of the library do not need it and so that a host
// process that already carries its own libnccl (e.g. PyTorch's) keeps using that one.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/ybgpu_compaction.h"
#include "dev_logic.cuh"
#include "host_sst.h"
#include "range_plan.h"

namespace {

using namespace ybgpu::plan;

struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*GetVersion)(int*) = nullptr;
};

const NcclApi* Nccl(std::string* err) {
  static NcclApi api;
  static std::once_flag once;
  static std::string load_err;
  std::call_once(once, [] {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);        // the copy the process already has
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) { load_err = std::string("cannot load libnccl: ") + dlerror(); return; }
    api.handle = h;
#define YB_SYM(field, name)                                                            \
    *reinterpret_cast<void**>(&api.field) = dlsym(h, name);                            \
    if (!api.field) { load_err = std::string("libnccl lacks ") + name; api.handle = nullptr; return; }
    YB_SYM(GetUniqueId, "ncclGetUniqueId") YB_SYM(CommInitRank, "ncclCommInitRank") YB_SYM(CommDestroy, "ncclCommDestroy")
    YB_SYM(Send, "ncclSend") YB_SYM(Recv, "ncclRecv") YB_SYM(AllGather, "ncclAllGather") YB_SYM(GroupStart, "ncclGroupStart")
    YB_SYM(GroupEnd, "ncclGroupEnd") YB_SYM(GetErrorString, "ncclGetErrorString") YB_SYM(GetVersion, "ncclGetVersion")
#undef YB_SYM
  });
  if (!api.handle) { if (err) *err = load_err; return nullptr; }
  return &api;
}

}  // namespace

struct ybgpu_range_comm {
  ncclComm_t comm = nullptr;
  int rank = 0, world = 1, device = 0;
  cudaStream_t stream = nullptr;         // collectives
  cudaStream_t copy_stream = nullptr;    // host -> device staging
  int nccl_version = 0;
};

namespace {

#define RX_CUDA(expr)                                                                                          \
  do { cudaError_t _e = (expr); if (_e != cudaSuccess) return fail(YBGPU_RUNTIME_ERROR, std::string(#expr) + ": " + cudaGetErrorString(_e)); } while (0)
#define RX_NCCL(expr)                                                                                          \
  do { ncclResult_t _r = (expr); if (_r != ncclSuccess) return fail(YBGPU_RUNTIME_ERROR, std::string(#expr) + ": " + N->GetErrorString(_r)); } while (0)

struct DevBuf {
  void* p = nullptr;
  ~DevBuf() { if (p) cudaFree(p); }
  cudaError_t Alloc(size_t n) { if (p) cudaFree(p); p = nullptr; return cudaMalloc(&p, std::max<size_t>(n, 16)); }
  uint8_t* u8() const { return static_cast<uint8_t*>(p); }
};

// Variable-size host blobs, one per rank, gathered on every rank: sizes first, then the bytes padded to the longest.
ybgpu_status AllGatherBlobs(ybgpu_range_comm* c, const NcclApi* N, const std::string& mine, std::vector<std::string>* all, std::string* err) {
  auto fail = [&](ybgpu_status s, const std::string& m) { *err = m; return s; };
  const int W = c->world;
  DevBuf d_sz, d_all_sz;
  RX_CUDA(d_sz.Alloc(8)); RX_CUDA(d_all_sz.Alloc(8 * W));
  const uint64_t my_size = mine.size();
  RX_CUDA(cudaMemcpyAsync(d_sz.p, &my_size, 8, cudaMemcpyHostToDevice, c->stream));
  RX_NCCL(N->AllGather(d_sz.p, d_all_sz.p, 8, ncclUint8, c->comm, c->stream));
  std::vector<uint64_t> sizes(W);
  RX_CUDA(cudaMemcpyAsync(sizes.data(), d_all_sz.p, 8 * W, cudaMemcpyDeviceToHost, c->stream));
  RX_CUDA(cudaStreamSynchronize(c->stream));
  uint64_t mx = 0;
  for (uint64_t s : sizes) mx = std::max(mx, s);
  mx = (mx + 15) & ~15ull;
  all->assign(W, std::string());
  if (mx == 0) return YBGPU_OK;
  DevBuf d_mine, d_all;
  RX_CUDA(d_mine.Alloc(mx)); RX_CUDA(d_all.Alloc(mx * W));
  RX_CUDA(cudaMemsetAsync(d_mine.p, 0, mx, c->stream));
  if (!mine.empty()) RX_CUDA(cudaMemcpyAsync(d_mine.p, mine.data(), mine.size(), cudaMemcpyHostToDevice, c->stream));
  RX_NCCL(N->AllGather(d_mine.p, d_all.p, mx, ncclUint8, c->comm, c->stream));
  std::string host(mx * W, '\0');
  RX_CUDA(cudaMemcpyAsync(&host[0], d_all.p, mx * W, cudaMemcpyDeviceToHost, c->stream));
  RX_CUDA(cudaStreamSynchronize(c->stream));
  for (int r = 0; r < W; r++) (*all)[r].assign(host, static_cast<size_t>(r) * mx, sizes[r]);
  return YBGPU_OK;
}

void PutU32(std::string* s, uint32_t v) { s->append(reinterpret_cast<const char*>(&v), 4); }
void PutU64(std::string* s, uint64_t v) { s->append(reinterpret_cast<const char*>(&v), 8); }
struct Reader {
  const char* p; const char* e; bool ok = true;
  uint32_t U32() { uint32_t v = 0; if (e - p < 4) { ok = false; return 0; } memcpy(&v, p, 4); p += 4; return v; }
  uint64_t U64() { uint64_t v = 0; if (e - p < 8) { ok = false; return 0; } memcpy(&v, p, 8); p += 8; return v; }
  std::string Bytes(size_t n) { if (static_cast<size_t>(e - p) < n) { ok = false; return std::string(); } std::string r(p, n); p += n; return r; }
};

// One contiguous run of data blocks of a source file, as it travels: [16 zero bytes][blocks + trailers][pad to 16][16 zero bytes]
struct Slice {
  uint32_t file = 0;                 // source-local file index (sender) / running index (receiver)
  size_t a = 0, b = 0;               // blocks [a, b) of the source file (sender only)
  uint64_t src_off = 0, bytes = 0;   // byte span inside the source file
  uint64_t framed = 0;               // bytes on the wire
  int32_t key_encoding = 1;
  uint64_t ht_filter = YBGPU_HT_INVALID;
  std::vector<ybgpu_block_handle> handles;     // offsets relative to the slice (receiver)
  uint64_t recv_off = 0;             // where the slice's first block byte lies in the receive buffer of its source
};

}  // namespace

extern "C" {

ybgpu_status ybgpu_range_comm_unique_id(uint8_t id[128]) {
  std::string err;
  const NcclApi* N = Nccl(&err);
  if (!N || !id) return YBGPU_RUNTIME_ERROR;
  static_assert(sizeof(ncclUniqueId) <= 128, "ncclUniqueId");
  ncclUniqueId u;
  if (N->GetUniqueId(&u) != ncclSuccess) return YBGPU_RUNTIME_ERROR;
  memset(id, 0, 128);
  memcpy(id, &u, sizeof(u));
  return YBGPU_OK;
}

ybgpu_status ybgpu_range_comm_create(const uint8_t id[128], int32_t rank, int32_t world, int32_t device, ybgpu_range_comm** out) {
  std::string err;
  const NcclApi* N = Nccl(&err);
  if (!N || !id || !out || world < 1 || rank < 0 || rank >= world) return YBGPU_INVALID_ARGUMENT;
  if (cudaSetDevice(device) != cudaSuccess) return YBGPU_RUNTIME_ERROR;
  std::unique_ptr<ybgpu_range_comm> c(new ybgpu_range_comm);
  c->rank = rank; c->world = world; c->device = device;
  ncclUniqueId u;
  memcpy(&u, id, sizeof(u));
  if (N->CommInitRank(&c->comm, world, u, rank) != ncclSuccess) return YBGPU_RUNTIME_ERROR;
  if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) return YBGPU_RUNTIME_ERROR;
  if (cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking) != cudaSuccess) return YBGPU_RUNTIME_ERROR;
  N->GetVersion(&c->nccl_version);
  if (rank == 0)
    fprintf(stderr, "[ybgpu] range communicator: %d ranks, NCCL %d.%d.%d, device %d\n", world, c->nccl_version / 10000,
            (c->nccl_version / 100) % 100, c->nccl_version % 100, device);
  *out = c.release();
  return YBGPU_OK;
}

void ybgpu_range_comm_destroy(ybgpu_range_comm* c) {
  if (!c) return;
  std::string err;
  const NcclApi* N = Nccl(&err);
  cudaSetDevice(c->device);
  if (c->stream) { cudaStreamSynchronize(c->stream); }
  if (N && c->comm) N->CommDestroy(c->comm);
  if (c->stream) cudaStreamDestroy(c->stream);
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  delete c;
}

ybgpu_status ybgpu_compact_range_sharded(ybgpu_range_comm* c, const ybgpu_job_options* options, const ybgpu_input_file* files,
                                         uint32_t num_files, uint32_t rounds, uint64_t chunk_bytes,
                                         uint8_t* data_out, uint64_t data_cap, uint8_t* meta_out, uint64_t meta_cap,
                                         ybgpu_range_shard_result* result, ybgpu_job_stats* total, char* err, uint64_t err_cap) {
  auto fail = [&](ybgpu_status s, const std::string& msg) {
    if (err && err_cap) snprintf(err, err_cap, "%s", msg.c_str());
    return s;
  };
  if (options && !ybgpu::host::OutputCompressionSupported(options->output_compression))
    return fail(YBGPU_NOT_SUPPORTED, ybgpu::host::UnsupportedOutputCompression(options->output_compression));
  std::string nerr;
  const NcclApi* N = Nccl(&nerr);
  if (!N) return fail(YBGPU_RUNTIME_ERROR, nerr);
  if (!c || !options || (!files && num_files) || !data_out || !meta_out || !result) return fail(YBGPU_INVALID_ARGUMENT, "null argument");
  if (options->range_lower_len || options->range_upper_len) return fail(YBGPU_INVALID_ARGUMENT, "range bounds are set by the planner");
  for (uint32_t f = 0; f < num_files; f++)
    if (files[f].num_cotable_filters) return fail(YBGPU_NOT_SUPPORTED, "per-database cotable HybridTime filters do not travel with the exchanged block slices");
  if (rounds == 0) rounds = 1;
  if (chunk_bytes == 0) chunk_bytes = 64ull << 20;
  chunk_bytes = (chunk_bytes + 15) & ~15ull;
  memset(result, 0, sizeof(*result));
  RX_CUDA(cudaSetDevice(c->device));
  const int W = c->world, me = c->rank;
  const uint32_t n_ranges_want = static_cast<uint32_t>(W) * rounds;
  const auto t_start = std::chrono::steady_clock::now();
  auto secs = [&]() { return std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count(); };

  // ---- 1. plan
  std::vector<ParsedInput> in;
  std::string perr;
  if (!ParseInputs(files, num_files, &in, &perr)) return fail(YBGPU_CORRUPTION, perr);
  std::string blob;                  // [largest user key][samples...]
  {
    std::string largest_local; bool have = false;
    for (uint32_t f = 0; f < num_files; f++) {
      std::string k;
      if (!LastKeyOfFile(files[f], in[f].meta, &k, options->verify_checksums != 0)) return fail(YBGPU_CORRUPTION, "cannot read the last key of input " + std::to_string(f));
      if (k.empty()) continue;
      const std::string u = UserPart(k);
      if (!have || largest_local < u) { largest_local = u; have = true; }
    }
    std::vector<Sample> samples;
    CollectSamples(in, std::max(1u, n_ranges_want / static_cast<uint32_t>(W)), &samples);
    PutU32(&blob, have ? 1 : 0); PutU32(&blob, static_cast<uint32_t>(largest_local.size())); blob += largest_local;
    PutU32(&blob, static_cast<uint32_t>(samples.size()));
    for (const Sample& s : samples) { PutU64(&blob, s.w); PutU32(&blob, static_cast<uint32_t>(s.key.size())); blob += s.key; }
  }
  std::vector<std::string> blobs;
  if (ybgpu_status s = AllGatherBlobs(c, N, blob, &blobs, &nerr)) return fail(s, nerr);
  std::string largest_user; bool have_largest = options->has_largest_user_key != 0;
  if (have_largest) largest_user.assign(reinterpret_cast<const char*>(options->largest_user_key), options->largest_user_key_len);
  std::vector<Sample> all_samples;
  for (const std::string& bl : blobs) {
    Reader r{bl.data(), bl.data() + bl.size()};
    const uint32_t has = r.U32(); const uint32_t ll = r.U32(); const std::string lk = r.Bytes(ll);
    if (has && !options->has_largest_user_key && (!have_largest || largest_user < lk)) { largest_user = lk; have_largest = true; }
    const uint32_t ns = r.U32();
    for (uint32_t i = 0; i < ns && r.ok; i++) { Sample s; s.w = r.U64(); const uint32_t kl = r.U32(); s.key = r.Bytes(kl); all_samples.push_back(std::move(s)); }
    if (!r.ok) return fail(YBGPU_CORRUPTION, "malformed planning blob");
  }
  const std::vector<std::string> splitters = SplittersFromSamples(std::move(all_samples), n_ranges_want, options->retention_enabled != 0);
  const uint32_t n_ranges = static_cast<uint32_t>(splitters.size()) + 1;      // <= n_ranges_want; trailing ranges may not exist
  auto range_lo = [&](uint32_t g) { return g == 0 ? std::string() : splitters[g - 1]; };
  auto range_hi = [&](uint32_t g) { return g + 1 >= n_ranges ? std::string() : splitters[g]; };
  result->num_ranges = n_ranges;
  result->plan_seconds = secs();

  // ---- per round: exchange + compact
  ybgpu::host::TableOptions topt;
  topt.block_size = options->block_size; topt.block_restart_interval = options->block_restart_interval;
  topt.block_size_deviation = options->block_size_deviation; topt.index_block_size = options->index_block_size;
  topt.min_keys_per_index_block = options->min_keys_per_index_block; topt.key_encoding = options->output_key_encoding;
  topt.filter_policy = options->filter_policy; if (options->filter_block_size) topt.filter_block_size = options->filter_block_size; topt.compression = options->output_compression;
  struct Piece { std::string meta, smallest, largest; uint64_t data_len = 0; };
  std::vector<Piece> pieces;
  ybgpu_job_stats tot; memset(&tot, 0, sizeof(tot));
  bool first_output = true;
  uint64_t data_used = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  RX_CUDA(cudaEventCreate(&ev0)); RX_CUDA(cudaEventCreate(&ev1));
  struct EvGuard { cudaEvent_t a, b; ~EvGuard() { cudaEventDestroy(a); cudaEventDestroy(b); } } evg{ev0, ev1};

  for (uint32_t t = 0; t < rounds; t++) {
    // the range of rank d in this round
    auto gidx = [&](int d) { return static_cast<uint32_t>(d) * rounds + t; };
    // ---- 2a. what I send to whom
    std::vector<std::vector<Slice>> send(W);
    std::vector<uint64_t> send_bytes(W, 0);
    std::vector<std::string> send_meta(W);
    for (int d = 0; d < W; d++) {
      const uint32_t g = gidx(d);
      if (g >= n_ranges) continue;
      const std::string lo = range_lo(g), hi = range_hi(g);
      std::vector<Span> spans;
      for (uint32_t f = 0; f < num_files; f++) {
        SpansForRange(in[f], lo, hi, options->retention_enabled != 0, &spans);
        const auto& blocks = in[f].meta.data_blocks;
        for (const Span& sp : spans) {
          Slice sl;
          sl.file = f; sl.a = sp.a; sl.b = sp.b;
          sl.src_off = blocks[sp.a].offset;
          sl.bytes = blocks[sp.b - 1].offset + blocks[sp.b - 1].size + 5 - sl.src_off;
          sl.framed = 16 + ((sl.bytes + 15) & ~15ull) + 16;
          sl.key_encoding = in[f].meta.key_encoding; sl.ht_filter = files[f].hybrid_time_filter;
          std::string& m = send_meta[d];
          PutU64(&m, sl.bytes); PutU64(&m, sl.framed); PutU32(&m, static_cast<uint32_t>(sl.key_encoding)); PutU64(&m, sl.ht_filter);
          PutU32(&m, static_cast<uint32_t>(sp.b - sp.a));
          for (size_t i = sp.a; i < sp.b; i++) { PutU64(&m, blocks[i].offset - sl.src_off); PutU64(&m, blocks[i].size); }
          send_bytes[d] += sl.framed;
          send[d].push_back(std::move(sl));
        }
      }
    }
    // ---- 2b. counts first: the byte matrix (data and handle bytes per pair) through one all-gather
    std::string row;
    for (int d = 0; d < W; d++) { PutU64(&row, send_bytes[d]); PutU64(&row, send_meta[d].size()); }
    std::vector<std::string> rows;
    if (ybgpu_status s = AllGatherBlobs(c, N, row, &rows, &nerr)) return fail(s, nerr);
    std::vector<uint64_t> recv_bytes(W, 0), recv_meta_bytes(W, 0);
    for (int src = 0; src < W; src++) {
      if (rows[src].size() != static_cast<size_t>(16 * W)) return fail(YBGPU_CORRUPTION, "malformed byte matrix");
      memcpy(&recv_bytes[src], rows[src].data() + 16 * me, 8);
      memcpy(&recv_meta_bytes[src], rows[src].data() + 16 * me + 8, 8);
    }
    RX_CUDA(cudaEventRecord(ev0, c->stream));
    // ---- 2c. handle lists (small): one grouped send / recv
    std::vector<std::string> recv_meta(W);
    {
      uint64_t sm = 0, rm = 0;
      std::vector<uint64_t> soff(W), roff(W);
      for (int d = 0; d < W; d++) { soff[d] = sm; sm += (send_meta[d].size() + 15) & ~15ull; roff[d] = rm; rm += (recv_meta_bytes[d] + 15) & ~15ull; }
      DevBuf d_s, d_r;
      RX_CUDA(d_s.Alloc(sm)); RX_CUDA(d_r.Alloc(rm));
      for (int d = 0; d < W; d++)
        if (!send_meta[d].empty()) RX_CUDA(cudaMemcpyAsync(d_s.u8() + soff[d], send_meta[d].data(), send_meta[d].size(), cudaMemcpyHostToDevice, c->stream));
      RX_NCCL(N->GroupStart());
      for (int p = 0; p < W; p++) {
        if (!send_meta[p].empty()) RX_NCCL(N->Send(d_s.u8() + soff[p], send_meta[p].size(), ncclUint8, p, c->comm, c->stream));
        if (recv_meta_bytes[p]) RX_NCCL(N->Recv(d_r.u8() + roff[p], recv_meta_bytes[p], ncclUint8, p, c->comm, c->stream));
      }
      RX_NCCL(N->GroupEnd());
      for (int p = 0; p < W; p++) {
        recv_meta[p].resize(recv_meta_bytes[p]);
        if (recv_meta_bytes[p]) RX_CUDA(cudaMemcpyAsync(&recv_meta[p][0], d_r.u8() + roff[p], recv_meta_bytes[p], cudaMemcpyDeviceToHost, c->stream));
      }
      RX_CUDA(cudaStreamSynchronize(c->stream));
    }
    // ---- 2d. the data: receive buffers in HBM (one per source), staging for what I send, chunk by chunk
    std::vector<DevBuf> rbuf(W);
    uint64_t recv_total = 0;
    for (int p = 0; p < W; p++) { if (recv_bytes[p]) { RX_CUDA(rbuf[p].Alloc(recv_bytes[p] + 64)); recv_total += recv_bytes[p]; } }
    uint64_t send_total = 0, max_pair = 0;
    for (int p = 0; p < W; p++) { send_total += send_bytes[p]; max_pair = std::max(max_pair, std::max(send_bytes[p], recv_bytes[p])); }
    {
      // every rank must run the same number of chunk rounds: the longest stream of the whole matrix
      uint64_t global_max = 0;
      for (int src = 0; src < W; src++)
        for (int d = 0; d < W; d++) { uint64_t v; memcpy(&v, rows[src].data() + 16 * d, 8); global_max = std::max(global_max, v); }
      const uint64_t n_chunks = (global_max + chunk_bytes - 1) / chunk_bytes;
      DevBuf stage[2];
      if (send_total) { RX_CUDA(stage[0].Alloc(chunk_bytes * W)); RX_CUDA(stage[1].Alloc(chunk_bytes * W)); }
      cudaEvent_t staged[2] = {nullptr, nullptr}, sent[2] = {nullptr, nullptr};
      for (int i = 0; i < 2; i++) { RX_CUDA(cudaEventCreateWithFlags(&staged[i], cudaEventDisableTiming)); RX_CUDA(cudaEventCreateWithFlags(&sent[i], cudaEventDisableTiming)); }
      struct EvG2 { cudaEvent_t* a; cudaEvent_t* b; ~EvG2() { for (int i = 0; i < 2; i++) { cudaEventDestroy(a[i]); cudaEventDestroy(b[i]); } } } evg2{staged, sent};
      // stages chunk q of every destination's stream into stage[q & 1] on the copy stream
      auto stage_chunk = [&](uint64_t q) -> cudaError_t {
        const int sb = static_cast<int>(q & 1);
        if (q >= 2) { cudaError_t e = cudaStreamWaitEvent(c->copy_stream, sent[sb], 0); if (e != cudaSuccess) return e; }   // its previous content has left
        for (int d = 0; d < W; d++) {
          const uint64_t lo = q * chunk_bytes, hi = std::min(send_bytes[d], lo + chunk_bytes);
          if (lo >= hi) continue;
          uint8_t* dst = stage[sb].u8() + static_cast<size_t>(d) * chunk_bytes;
          cudaError_t e = cudaMemsetAsync(dst, 0, hi - lo, c->copy_stream);           // frames and pads are zeros
          if (e != cudaSuccess) return e;
          uint64_t pos = 0;                                                           // stream position of the slice frame
          for (const Slice& sl : send[d]) {
            const uint64_t b0 = pos + 16, b1 = b0 + sl.bytes;                        // the slice's block bytes in the stream
            const uint64_t x0 = std::max(b0, lo), x1 = std::min(b1, hi);
            if (x0 < x1) {
              e = cudaMemcpyAsync(dst + (x0 - lo), files[sl.file].data_file + sl.src_off + (x0 - b0), x1 - x0, cudaMemcpyHostToDevice, c->copy_stream);
              if (e != cudaSuccess) return e;
            }
            pos += sl.framed;
            if (pos >= hi) break;
          }
        }
        return cudaEventRecord(staged[sb], c->copy_stream);
      };
      if (n_chunks && send_total) RX_CUDA(stage_chunk(0));
      for (uint64_t q = 0; q < n_chunks; q++) {
        const int sb = static_cast<int>(q & 1);
        if (send_total && q + 1 < n_chunks) RX_CUDA(stage_chunk(q + 1));              // next chunk travels H2D while this one is on NVLink
        if (send_total) RX_CUDA(cudaStreamWaitEvent(c->stream, staged[sb], 0));
        RX_NCCL(N->GroupStart());
        for (int p = 0; p < W; p++) {
          const uint64_t lo = q * chunk_bytes;
          const uint64_t shi = std::min(send_bytes[p], lo + chunk_bytes), rhi = std::min(recv_bytes[p], lo + chunk_bytes);
          if (lo < shi) RX_NCCL(N->Send(stage[sb].u8() + static_cast<size_t>(p) * chunk_bytes, shi - lo, ncclUint8, p, c->comm, c->stream));
          if (lo < rhi) RX_NCCL(N->Recv(rbuf[p].u8() + lo, rhi - lo, ncclUint8, p, c->comm, c->stream));
        }
        RX_NCCL(N->GroupEnd());
        if (send_total) RX_CUDA(cudaEventRecord(sent[sb], c->stream));
      }
      RX_CUDA(cudaEventRecord(ev1, c->stream));
      RX_CUDA(cudaStreamSynchronize(c->stream));
      RX_CUDA(cudaStreamSynchronize(c->copy_stream));
    }
    float ms = 0;
    RX_CUDA(cudaEventElapsedTime(&ms, ev0, ev1));
    result->exchange_seconds += ms / 1e3;
    result->sent_bytes += send_total; result->received_bytes += recv_total;
    result->sent_to_peers_bytes += send_total - send_bytes[me];

    // ---- 3. compact my range of this round
    const uint32_t g = gidx(me);
    if (g >= n_ranges) continue;
    const std::string lo = range_lo(g), hi = range_hi(g);
    ybgpu_job_options o = *options;
    o.device = c->device;
    o.cuda_stream = YBGPU_STREAM_PRIVATE;
    o.range_lower = reinterpret_cast<const uint8_t*>(lo.data()); o.range_lower_len = lo.size();
    o.range_upper = reinterpret_cast<const uint8_t*>(hi.data()); o.range_upper_len = hi.size();
    o.has_largest_user_key = have_largest ? 1 : 0;
    o.largest_user_key = reinterpret_cast<const uint8_t*>(largest_user.data()); o.largest_user_key_len = largest_user.size();
    ybgpu_job* job = nullptr;
    ybgpu_status s = ybgpu_job_create(&o, &job);
    if (s != YBGPU_OK) return fail(s, std::string("create: ") + ybgpu_last_error());
    struct JobGuard { ybgpu_job* j; ~JobGuard() { if (j) ybgpu_job_destroy(j); } } jg{job};
    uint32_t added = 0;
    for (int p = 0; p < W; p++) {
      Reader r{recv_meta[p].data(), recv_meta[p].data() + recv_meta[p].size()};
      uint64_t pos = 0;
      while (r.p < r.e) {
        const uint64_t bytes = r.U64(), framed = r.U64(); const uint32_t enc = r.U32(); const uint64_t htf = r.U64(); const uint32_t nb = r.U32();
        std::vector<ybgpu_block_handle> h(nb);
        for (uint32_t i = 0; i < nb; i++) { h[i].offset = r.U64(); h[i].size = r.U64(); }
        if (!r.ok || pos + framed > recv_bytes[p]) return fail(YBGPU_CORRUPTION, "malformed slice list from rank " + std::to_string(p));
        s = ybgpu_job_add_input_device(job, rbuf[p].u8() + pos + 16, bytes, h.data(), nb, static_cast<int32_t>(enc), htf);
        if (s != YBGPU_OK) return fail(s, std::string("add_input_device: ") + ybgpu_job_error(job));
        pos += framed;
        added++;
      }
    }
    if (!added) continue;
    s = ybgpu_job_run(job, nullptr);
    if (s != YBGPU_OK) return fail(s, std::string("run (range ") + std::to_string(g) + "): " + ybgpu_job_error(job));
    uint64_t dl = 0, ml = 0;
    s = ybgpu_job_output_sizes(job, &dl, &ml);
    if (s != YBGPU_OK) return fail(s, std::string("output_sizes: ") + ybgpu_job_error(job));
    ybgpu_job_stats st;
    if (dl) {
      if (data_used + dl > data_cap) return fail(YBGPU_INVALID_ARGUMENT, "output buffer too small");
      Piece pc;
      pc.meta.resize(ml);
      s = ybgpu_job_fetch_output(job, data_out + data_used, dl, reinterpret_cast<uint8_t*>(&pc.meta[0]), ml);
      if (s != YBGPU_OK) return fail(s, std::string("fetch_output: ") + ybgpu_job_error(job));
      uint8_t sk[4096], lk[4096]; uint64_t sl = 0, ll = 0;
      s = ybgpu_job_output_boundaries(job, sk, &sl, lk, &ll);
      if (s != YBGPU_OK) return fail(s, std::string("output_boundaries: ") + ybgpu_job_error(job));
      pc.smallest.assign(reinterpret_cast<char*>(sk), sl); pc.largest.assign(reinterpret_cast<char*>(lk), ll);
      pc.data_len = dl;
      data_used += dl;
      pieces.push_back(std::move(pc));
    }
    ybgpu_job_get_stats(job, &st);
    tot.num_input_records += st.num_input_records; tot.num_output_records += st.num_output_records;
    tot.num_record_drop_hidden += st.num_record_drop_hidden; tot.num_record_drop_obsolete += st.num_record_drop_obsolete;
    tot.num_record_drop_feed += st.num_record_drop_feed;
    tot.total_input_raw_key_bytes += st.total_input_raw_key_bytes; tot.total_input_raw_value_bytes += st.total_input_raw_value_bytes;
    tot.total_output_raw_key_bytes += st.total_output_raw_key_bytes; tot.total_output_raw_value_bytes += st.total_output_raw_value_bytes;
    tot.num_output_data_blocks += st.num_output_data_blocks;
    if (st.num_output_records) {
      tot.smallest_seqno = first_output ? st.smallest_seqno : std::min(tot.smallest_seqno, st.smallest_seqno);
      tot.largest_seqno = std::max(tot.largest_seqno, st.largest_seqno);
      first_output = false;
    }
    tot.gpu_seconds += st.gpu_seconds; tot.gpu_kernel_launches += st.gpu_kernel_launches;
    tot.h2d_bytes += st.h2d_bytes; tot.d2h_bytes += st.d2h_bytes;
    for (int i = 0; i < 8; i++) { tot.phase_seconds[i] += st.phase_seconds[i]; tot.phase_launches[i] += st.phase_launches[i]; }
    tot.path_flags |= st.path_flags; tot.tiles_inside_rows += st.tiles_inside_rows;
  }

  // ---- 4. this rank's table
  result->data_len = data_used;
  result->num_pieces = static_cast<uint32_t>(pieces.size());
  if (!pieces.empty()) {
    std::string meta;
    if (pieces.size() == 1) meta.swap(pieces[0].meta);
    else {
      ybgpu::host::ConcatBuilder cb(topt);
      for (size_t i = 0; i < pieces.size(); i++) {
        ybgpu::host::SstPiece a, nx;
        a.meta = reinterpret_cast<const uint8_t*>(pieces[i].meta.data()); a.meta_len = pieces[i].meta.size(); a.data_len = pieces[i].data_len;
        a.smallest = pieces[i].smallest; a.largest = pieces[i].largest;
        if (i + 1 < pieces.size()) { nx.smallest = pieces[i + 1].smallest; nx.largest = pieces[i + 1].largest; }
        const std::string e = cb.AddPiece(a, i + 1 < pieces.size() ? &nx : nullptr);
        if (!e.empty()) return fail(YBGPU_INVALID_ARGUMENT, "assembly: " + e);
      }
      const std::string e = cb.Finish(&meta);
      if (!e.empty()) return fail(YBGPU_INVALID_ARGUMENT, "assembly: " + e);
    }
    if (meta.size() > meta_cap) return fail(YBGPU_INVALID_ARGUMENT, "metadata buffer too small");
    memcpy(meta_out, meta.data(), meta.size());
    result->meta_len = meta.size();
    result->smallest_key_len = static_cast<uint32_t>(std::min<size_t>(pieces.front().smallest.size(), sizeof(result->smallest_key)));
    result->largest_key_len = static_cast<uint32_t>(std::min<size_t>(pieces.back().largest.size(), sizeof(result->largest_key)));
    memcpy(result->smallest_key, pieces.front().smallest.data(), result->smallest_key_len);
    memcpy(result->largest_key, pieces.back().largest.data(), result->largest_key_len);
  }
  {
    const uint32_t g0 = static_cast<uint32_t>(me) * rounds, g1 = std::min(n_ranges, g0 + rounds);
    if (g0 < n_ranges) {
      const std::string lo = range_lo(g0), hi = range_hi(g1 - 1);
      result->range_lower_len = static_cast<uint32_t>(lo.size()); memcpy(result->range_lower, lo.data(), lo.size());
      result->range_upper_len = static_cast<uint32_t>(hi.size()); memcpy(result->range_upper, hi.data(), hi.size());
    }
  }
  result->total_seconds = secs();
  tot.output_data_file_size = result->data_len; tot.output_meta_file_size = result->meta_len;
  if (total) *total = tot;
  return YBGPU_OK;
}

}  // extern "C"
