// engine.cu — H100 (sm_90a) DocDB compaction engine: kernels + host orchestration.
//
// Pipeline (one ybgpu_job = one rocksdb::CompactionJob::Run, reference
// src/yb/rocksdb/db/compaction_job.cc:664-895):
//
//   K1  k_prepass   per data block: entry count, max key length, raw sizes        (BlockIter walk,
//   K1' k_decode    per restart interval: delta-decode keys -> fixed-stride records  table/block.cc:348-447)
//   K2  k_sample_*  DocKey-aligned multiway partition of the k sorted runs into tiles
//   K3  k_merge_filter  per tile: rank-based k-way merge in shared memory (MergingIterator,
//                   table/merger.cc), CompactionIterator rule A + seqno zeroing
//                   (db/compaction_iterator.cc:388-400,467-483) and the DocDB retention
//                   predicate (docdb/docdb_compaction_context.cc:941-1311) per row group
//   K4  k_emit_*    scan survivors, gather keys + values into the output KV stream
//
// All byte/integer work, HBM-bound: no tensor cores. See DESIGN.md for the data layout and the
// per-kernel algorithmic bytes.
#include "engine.h"
#include "host_sst.h"

#include <cuda_runtime.h>
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <chrono>
#include <cstdlib>
#include <mutex>

namespace ybgpu {

#define CUDA_TRY(expr)                                                                      \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess) {                                                                \
      return FailCuda(#expr, _e);                                                           \
    }                                                                                       \
  } while (0)

// ---------------------------------------------------------------------------------------------
// Device-side views
struct RunView {
  const uint8_t* data;          // data file bytes (HBM)
  const uint64_t* blk_off;      // per data block
  const uint32_t* blk_size;
  uint32_t* blk_count;          // entries per block (K1), then exclusive prefix (blk_base)
  uint8_t* rec;                 // n_entries * S key records (K1')
  uint64_t* val_off;            // value offset inside `data` per entry
  uint32_t* val_crc;            // RAW CRC32C (zero initial register, no complement) of every entry's value bytes
  uint32_t nb;
  uint32_t n_entries;
  uint32_t restart_interval;    // entries per restart interval in this file
  uint32_t gid_base;            // global entry id of entry 0
  uint32_t key_encoding;        // rocksdb::KeyValueEncodingFormat of this file's data blocks
  uint64_t ht_filter;
  const uint32_t* cf_oid;       // per-database cotable HybridTime filters of the file: sorted database oids,
  const uint64_t* cf_ht;        //   their hybrid times (device arrays), and how many (0 = none)
  uint32_t cf_n;
};

struct JobDev {                 // device-global job state
  int error;                    // first DevError
  uint32_t error_where;         // block / tile index
  uint32_t max_ikey_len;        // K1
  uint32_t restart_interval[MAX_RUNS];
  unsigned long long in_key_bytes, in_val_bytes;
  unsigned long long n_counted, n_hidden, n_obsolete, n_feed_dropped, n_kept, out_key_bytes, out_val_bytes;
  unsigned long long min_seq, max_seq, n_kept_deletions;
  uint32_t n_rewrites;
  uint32_t n_tiles;
  uint32_t max_tile;            // largest tile of the current partition (k_tile_check)
  int ingest_fallback;          // k_ingest met something it does not take: the host runs the general kernels
  uint32_t n_compressed;        // compressed input blocks (Snappy, LZ4, LZ4HC) seen by k_restart_probe
  uint32_t n_lz4;               // ... of which LZ4 or LZ4HC
  uint32_t n_cont_tiles;        // merge tiles that started inside a row group
  unsigned long long digest;
  unsigned long long verify_fail; // output check: verify_pack() of the first failure, lowest (block, entry) wins; ~0 = none
};

struct JobParams {
  int S;                        // record stride
  int k;                        // number of runs
  int bottommost;
  uint64_t last_sequence;
  uint32_t largest_len; uint8_t largest[1024];   // Compaction::GetLargestUserKey
  uint32_t tile_cap;            // records per tile
  uint32_t H;                   // target rank step between tile boundaries
  uint32_t M;                   // sample stride
  RetentionDev R;
  RangeDev range;
};

struct Desc {                   // one per input entry in merged order
  uint32_t gid;
  uint32_t vlen_out;
  uint16_t klen;                // internal key length
  uint8_t flags;                // ENT_*
  uint8_t run;
  uint32_t rewrite_slot;
};

__device__ __forceinline__ void dev_fail(JobDev* J, int code, uint32_t where) {
  if (atomicCAS(&J->error, 0, code) == 0) J->error_where = where;
}

__device__ __forceinline__ uint32_t ldg_u32_unaligned(const uint8_t* p) {
  return static_cast<uint32_t>(p[0]) | (static_cast<uint32_t>(p[1]) << 8) | (static_cast<uint32_t>(p[2]) << 16) |
         (static_cast<uint32_t>(p[3]) << 24);
}

// ---------------------------------------------------------------------------------------------
// K1: one warp per data block, one lane per restart interval. Walks entry headers only.
__global__ void __launch_bounds__(256) k_prepass(const RunView* runs, const uint32_t* blk_base /*[k+1]*/, int k, JobDev* J) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  unsigned long long key_bytes = 0, val_bytes = 0;
  uint32_t max_klen = 0;
  const uint32_t total_blocks = blk_base[k];
  for (uint32_t gb = warp; gb < total_blocks; gb += nwarps) {
    int run_idx = 0;
    while (blk_base[run_idx + 1] <= gb) run_idx++;
    const RunView& run = runs[run_idx];
    const uint32_t b = gb - blk_base[run_idx];
    const uint8_t* blk = run.data + run.blk_off[b];
    const uint32_t size = run.blk_size[b];
    uint32_t count = 0;
    bool bad = false;
    uint32_t num_restarts = 0, restarts_off = 0;
    if (size < 4) bad = true;
    else {
      num_restarts = ldg_u32_unaligned(blk + size - 4);
      if (num_restarts == 0 || static_cast<uint64_t>(num_restarts) * 4 + 4 > size) bad = true;
      else restarts_off = size - 4 - 4 * num_restarts;
    }
    if (bad) { if (lane == 0) dev_fail(J, DEV_ERR_BAD_BLOCK, b); continue; }
    if (blk[size] != 0) { if (lane == 0) dev_fail(J, DEV_ERR_COMPRESSED, b); continue; }   // trailer type byte
    for (uint32_t r = lane; r < num_restarts; r += 32) {
      uint32_t p = ldg_u32_unaligned(blk + restarts_off + 4 * r);
      const uint32_t end = (r + 1 < num_restarts) ? ldg_u32_unaligned(blk + restarts_off + 4 * (r + 1)) : restarts_off;
      if (p > end || end > restarts_off) { dev_fail(J, DEV_ERR_BAD_BLOCK, b); break; }
      uint32_t n = 0, klen = 0;
      while (p < end) {
        uint32_t shared, non_shared, vlen;
        if (run.key_encoding == 2) {
          TspHeader th; uint32_t nk, ms, ml;
          int h = parse_entry_header_tsp(blk + p, end - p, &th);
          if (!h || (n == 0 && th.something_shared) || !tsp_key_layout(th, klen, &nk, &ms, &ml) ||
              static_cast<uint64_t>(p) + h + th.ns1 + th.ns2 + th.vlen > end) { dev_fail(J, DEV_ERR_BAD_ENTRY, b); n = 0; break; }
          klen = nk;
          if (klen < 8) { dev_fail(J, DEV_ERR_SHORT_KEY, b); break; }
          max_klen = max(max_klen, klen);
          p += h + th.ns1 + th.ns2 + th.vlen;
          n++;
          continue;
        }
        int h = parse_entry_header(blk + p, end - p, &shared, &non_shared, &vlen);
        if (!h || shared > klen || (n == 0 && shared != 0) ||
            static_cast<uint64_t>(p) + h + non_shared + vlen > end) { dev_fail(J, DEV_ERR_BAD_ENTRY, b); n = 0; break; }
        klen = shared + non_shared;
        if (klen < 8) { dev_fail(J, DEV_ERR_SHORT_KEY, b); break; }
        max_klen = max(max_klen, klen);
        key_bytes += klen; val_bytes += vlen;
        p += h + non_shared + vlen;
        n++;
      }
      count += n;
      // every interval but the last of a block must be full (BlockBuilder restarts every
      // block_restart_interval entries, table/block_builder.cc:357-361)
      uint32_t expect = __ldcg(&J->restart_interval[run_idx]);
      if (r + 1 < num_restarts) {
        if (expect == 0) { uint32_t old = atomicCAS(&J->restart_interval[run_idx], 0u, n); expect = old ? old : n; }
        if (expect != n) dev_fail(J, DEV_ERR_IRREGULAR_RESTARTS, b);
      } else if (expect != 0 && n > expect) {
        dev_fail(J, DEV_ERR_IRREGULAR_RESTARTS, b);
      }
    }
    for (int o = 16; o; o >>= 1) count += __shfl_xor_sync(0xffffffffu, count, o);
    if (lane == 0) run.blk_count[b] = count;
  }
  for (int o = 16; o; o >>= 1) {
    key_bytes += __shfl_xor_sync(0xffffffffu, key_bytes, o);
    val_bytes += __shfl_xor_sync(0xffffffffu, val_bytes, o);
    max_klen = max(max_klen, __shfl_xor_sync(0xffffffffu, max_klen, o));
  }
  (void)key_bytes; (void)val_bytes;
  if (lane == 0 && max_klen) atomicMax(&J->max_ikey_len, max_klen);
}

// Exclusive scan of a u32 array with one CTA (n up to a few million: nb per file).
__device__ __forceinline__ void scan_u32_cta(uint32_t* a, uint32_t n, uint32_t* total) {
  __shared__ uint32_t warp_sums[32];
  __shared__ uint32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (uint32_t base = 0; base < n; base += 1024) {
    uint32_t i = base + threadIdx.x;
    uint32_t v = i < n ? a[i] : 0;
    uint32_t x = v;
    for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) warp_sums[wid] = x;
    __syncthreads();
    if (wid == 0) {
      uint32_t w = warp_sums[lane];
      for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
      warp_sums[lane] = w;
    }
    __syncthreads();
    uint32_t excl = carry + (wid ? warp_sums[wid - 1] : 0) + x - v;
    if (i < n) a[i] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) carry += warp_sums[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry;
}
__global__ void __launch_bounds__(1024) k_scan_u32_single(uint32_t* a, uint32_t n, uint32_t* total) { scan_u32_cta(a, n, total); }
// Per-run exclusive scan of the per-block entry counts: CTA r scans run r.
__global__ void __launch_bounds__(1024) k_scan_blk_counts(const RunView* runs, uint32_t* totals) {
  scan_u32_cta(runs[blockIdx.x].blk_count, runs[blockIdx.x].nb, totals + blockIdx.x);
}

// K1' (single launch): all files at once. A warp takes DEC_WB consecutive data blocks of one file
// and spreads their restart intervals over its 32 lanes (a 32 KB block of 300-byte entries has only
// ~7 intervals, so one block per warp would leave most lanes idle).
constexpr int DEC_WB = 4;
template <int KMAX>
__global__ void __launch_bounds__(128) k_decode_all(const RunView* runs, const uint32_t* run_group_base /*[k+1]*/, int k, int S,
                                                   const RangeDev* range, JobDev* J) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  __align__(16) uint8_t keybuf[KMAX];
  const uint32_t total_groups = run_group_base[k];
  for (uint32_t g = warp; g < total_groups; g += nwarps) {
    int ri_ = 0;
    while (run_group_base[ri_ + 1] <= g) ri_++;
    const RunView& run = runs[ri_];
    const uint32_t b0 = (g - run_group_base[ri_]) * DEC_WB;
    const uint32_t nbk = min(static_cast<uint32_t>(DEC_WB), run.nb - b0);
    // restart counts of the group's blocks (lanes 0..nbk-1 read them), exclusive prefix by shuffles
    uint32_t nres = 0;
    if (lane < static_cast<int>(nbk)) {
      const uint8_t* blk = run.data + run.blk_off[b0 + lane];
      nres = ldg_u32_unaligned(blk + run.blk_size[b0 + lane] - 4);
    }
    uint32_t pre[DEC_WB + 1];
    pre[0] = 0;
#pragma unroll
    for (int q = 0; q < DEC_WB; q++) pre[q + 1] = pre[q] + __shfl_sync(0xffffffffu, nres, q);
    const uint32_t total_int = pre[DEC_WB];
    const uint32_t ri = run.restart_interval ? run.restart_interval : 1;
    for (uint32_t t = lane; t < total_int; t += 32) {
      int q = 0;
#pragma unroll
      for (int z = 1; z < DEC_WB; z++) if (t >= pre[z]) q = z;
      const uint32_t b = b0 + q, r = t - pre[q];
      const uint64_t boff = run.blk_off[b];
      const uint8_t* blk = run.data + boff;
      const uint32_t size = run.blk_size[b];
      const uint32_t num_restarts = pre[q + 1] - pre[q];
      const uint32_t restarts_off = size - 4 - 4 * num_restarts;
      uint32_t p = ldg_u32_unaligned(blk + restarts_off + 4 * r);
      const uint32_t end = (r + 1 < num_restarts) ? ldg_u32_unaligned(blk + restarts_off + 4 * (r + 1)) : restarts_off;
      uint32_t idx = run.blk_count[b] + r * ri;
      uint32_t prev_klen = 0;
      while (p < end) {
        uint32_t shared, non_shared, vlen, klen;
        if (run.key_encoding == 2) {
          // kKeyDeltaEncodingThreeSharedParts (table/block.cc:294-343, db/dbformat.h:413-470)
          TspHeader th; uint32_t ms, ml;
          int h = parse_entry_header_tsp(blk + p, end - p, &th);
          if (!h || !tsp_key_layout(th, prev_klen, &klen, &ms, &ml)) break;      // validated by k_prepass
          p += h;
          if (klen > KMAX) { dev_fail(J, DEV_ERR_KEY_TOO_LONG, b); break; }
          if (!th.something_shared) {
            for (uint32_t i = 0; i < th.ns1; i++) keybuf[i] = blk[p + i];
          } else {
            __align__(16) uint8_t tmp[KMAX];
            uint64_t last = 0;
            if (th.last_size) { for (int i = 7; i >= 0; i--) last = (last << 8) | keybuf[prev_klen - 8 + i]; last += th.last_inc; }
            uint32_t n2 = th.shared_prefix;
            for (uint32_t i = 0; i < th.ns1; i++) tmp[n2++] = blk[p + i];
            for (uint32_t i = 0; i < ml; i++) tmp[n2++] = keybuf[ms + i];
            for (uint32_t i = 0; i < th.ns2; i++) tmp[n2++] = blk[p + th.ns1 + i];
            if (th.last_size) for (int i = 0; i < 8; i++) tmp[n2++] = static_cast<uint8_t>(last >> (8 * i));
            for (uint32_t i = th.shared_prefix; i < klen; i++) keybuf[i] = tmp[i];
          }
          p += th.ns1 + th.ns2;
          vlen = th.vlen;
        } else {
          int h = parse_entry_header(blk + p, end - p, &shared, &non_shared, &vlen);
          if (!h) break;                                  // validated by k_prepass
          p += h;
          klen = shared + non_shared;
          if (klen > KMAX) { dev_fail(J, DEV_ERR_KEY_TOO_LONG, b); break; }
          for (uint32_t i = 0; i < non_shared; i++) keybuf[shared + i] = blk[p + i];
          p += non_shared;
        }
        prev_klen = klen;
        const uint32_t ulen = klen - 8;
        uint8_t* rec = run.rec + static_cast<size_t>(idx) * S;
        const int key_vecs = (S - 16) >> 4;
        for (int w = 0; w < key_vecs; w++) {
          uint4 v = *reinterpret_cast<const uint4*>(keybuf + 16 * w);
          const int valid = static_cast<int>(ulen) - 16 * w;
          uint32_t* vw = reinterpret_cast<uint32_t*>(&v);
#pragma unroll
          for (int c = 0; c < 4; c++) {
            const int vb = valid - 4 * c;
            if (vb <= 0) vw[c] = 0; else if (vb < 4) vw[c] &= (1u << (8 * vb)) - 1;
          }
          reinterpret_cast<uint4*>(rec)[w] = v;
        }
        uint64_t suffix = 0;
        for (int i = 7; i >= 0; i--) suffix = (suffix << 8) | keybuf[ulen + i];
        uint8_t flags = 0;
        if ((run.ht_filter != HT_FILTER_NONE || run.cf_n) && hidden_by_ht_filters(keybuf, ulen, run.ht_filter, run.cf_oid, run.cf_ht, run.cf_n))
          flags |= REC_F_HT_FILTERED;
        if (range && (range->lower_len | range->upper_len)) {
          if (range->lower_len && cmp_raw(keybuf, ulen, range->lower, range->lower_len) < 0) flags |= REC_F_OUT_OF_RANGE;
          if (range->upper_len && cmp_raw(keybuf, ulen, range->upper, range->upper_len) >= 0) flags |= REC_F_OUT_OF_RANGE;
        }
        const uint8_t vfirst = vlen ? blk[p] : 0;
        uint4 tr;
        tr.x = static_cast<uint32_t>(suffix); tr.y = static_cast<uint32_t>(suffix >> 32);
        tr.z = ulen | (static_cast<uint32_t>(vfirst) << 16) | (static_cast<uint32_t>(flags) << 24);
        tr.w = vlen;
        *reinterpret_cast<uint4*>(rec + S - 16) = tr;
        run.val_off[idx] = boff + p;
        p += vlen;
        idx++;
      }
    }
  }
}

// K1' fast path: shared-prefix inputs whose internal keys fit NVI 16-byte vectors, no per-file
// HybridTime filter, no key range. The previous internal key lives in registers (NVI uint4); an
// entry is decoded with at most NVI unaligned 16-byte fetches of its key delta, byte masks merge it
// over the shared prefix, and the record's key vectors are stored straight from the registers — no
// per-thread key buffer in local memory, no byte loops.
__device__ __forceinline__ uint32_t low_bytes_mask(int n) {   // 0xff in the first n bytes of a word, n in (-inf, +inf)
  return n <= 0 ? 0u : (n >= 4 ? 0xffffffffu : ((1u << (8 * n)) - 1u));
}
__device__ __forceinline__ uint4 low_bytes_mask16(int n) {    // same for a 16-byte vector
  return make_uint4(low_bytes_mask(n), low_bytes_mask(n - 4), low_bytes_mask(n - 8), low_bytes_mask(n - 12));
}
__device__ __forceinline__ uint4 ldg_unaligned16(const uint8_t* src) {   // reads [src & ~15, (src & ~15) + 32)
  const uint32_t sh = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(src) & 15);
  const uint4* sa = reinterpret_cast<const uint4*>(src - sh);
  const uint4 a = __ldg(sa);
  if (sh == 0) return a;
  const uint4 b = __ldg(sa + 1);
  uint32_t w0 = a.x, w1 = a.y, w2 = a.z, w3 = a.w, w4 = b.x, w5 = b.y, w6 = b.z, w7 = b.w;
  const uint32_t q = sh >> 2, bits = (sh & 3) * 8;
  if (q & 1) { w0 = w1; w1 = w2; w2 = w3; w3 = w4; w4 = w5; w5 = w6; w6 = w7; }
  if (q & 2) { w0 = w2; w1 = w3; w2 = w4; w3 = w5; w4 = w6; }
  return make_uint4(__funnelshift_r(w0, w1, bits), __funnelshift_r(w1, w2, bits), __funnelshift_r(w2, w3, bits), __funnelshift_r(w3, w4, bits));
}
template <int NVI>
__global__ void __launch_bounds__(128, 10) k_decode_fast(const RunView* runs, const uint32_t* run_group_base /*[k+1]*/, int k, int S, JobDev* J) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t total_groups = run_group_base[k];
  const int key_vecs = (S - 16) >> 4;                       // user-key vectors of a record (<= NVI)
  for (uint32_t g = warp; g < total_groups; g += nwarps) {
    int ri_ = 0;
    while (run_group_base[ri_ + 1] <= g) ri_++;
    const RunView& run = runs[ri_];
    const uint32_t b0 = (g - run_group_base[ri_]) * DEC_WB;
    const uint32_t nbk = min(static_cast<uint32_t>(DEC_WB), run.nb - b0);
    uint32_t nres = 0;
    if (lane < static_cast<int>(nbk)) {
      const uint8_t* blk = run.data + run.blk_off[b0 + lane];
      nres = ldg_u32_unaligned(blk + run.blk_size[b0 + lane] - 4);
    }
    uint32_t pre[DEC_WB + 1];
    pre[0] = 0;
#pragma unroll
    for (int q = 0; q < DEC_WB; q++) pre[q + 1] = pre[q] + __shfl_sync(0xffffffffu, nres, q);
    const uint32_t total_int = pre[DEC_WB];
    const uint32_t ri = run.restart_interval ? run.restart_interval : 1;
    for (uint32_t t = lane; t < total_int; t += 32) {
      int q = 0;
#pragma unroll
      for (int z = 1; z < DEC_WB; z++) if (t >= pre[z]) q = z;
      const uint32_t b = b0 + q, r = t - pre[q];
      const uint64_t boff = run.blk_off[b];
      const uint8_t* blk = run.data + boff;
      const uint32_t size = run.blk_size[b];
      const uint32_t num_restarts = pre[q + 1] - pre[q];
      const uint32_t restarts_off = size - 4 - 4 * num_restarts;
      uint32_t p = ldg_u32_unaligned(blk + restarts_off + 4 * r);
      const uint32_t end = (r + 1 < num_restarts) ? ldg_u32_unaligned(blk + restarts_off + 4 * (r + 1)) : restarts_off;
      uint32_t idx = run.blk_count[b] + r * ri;
      uint4 kv[NVI];                                          // previous internal key, zero beyond its length
#pragma unroll
      for (int w = 0; w < NVI; w++) kv[w] = make_uint4(0, 0, 0, 0);
      while (p < end) {
        uint32_t shared, non_shared, vlen;
        const int h = parse_entry_header(blk + p, end - p, &shared, &non_shared, &vlen);
        if (!h) break;                                        // validated by k_prepass
        p += h;
        const uint32_t klen = shared + non_shared;
        if (klen > 16 * NVI || klen < 8) { dev_fail(J, DEV_ERR_KEY_TOO_LONG, b); break; }
        const uint32_t ulen = klen - 8;
        // new internal key: bytes [0, shared) kept, [shared, klen) from the block, zero beyond
#pragma unroll
        for (int w = 0; w < NVI; w++) {
          const int lo = 16 * w;
          if (lo + 16 <= static_cast<int>(shared)) continue;
          if (lo >= static_cast<int>(klen)) { kv[w] = make_uint4(0, 0, 0, 0); continue; }
          const uint4 nw = ldg_unaligned16(blk + p + lo - static_cast<int>(shared));
          const uint4 keep = low_bytes_mask16(static_cast<int>(shared) - lo);
          const uint4 valid = low_bytes_mask16(static_cast<int>(klen) - lo);
          kv[w].x = (kv[w].x & keep.x) | (nw.x & ~keep.x & valid.x);
          kv[w].y = (kv[w].y & keep.y) | (nw.y & ~keep.y & valid.y);
          kv[w].z = (kv[w].z & keep.z) | (nw.z & ~keep.z & valid.z);
          kv[w].w = (kv[w].w & keep.w) | (nw.w & ~keep.w & valid.w);
        }
        p += non_shared;
        // suffix = internal-key bytes [ulen, ulen + 8): a 16-byte window starting at vector ulen / 16
        uint4 va = kv[0], vb = NVI > 1 ? kv[1] : make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int w = 1; w < NVI; w++) if (static_cast<int>(ulen >> 4) == w) { va = kv[w]; vb = (w + 1 < NVI) ? kv[w + 1] : make_uint4(0, 0, 0, 0); }
        uint32_t s0, s1;
        {
          uint32_t w0 = va.x, w1 = va.y, w2 = va.z, w3 = va.w, w4 = vb.x, w5 = vb.y;
          const uint32_t sh = ulen & 15, qq = sh >> 2, bits = (sh & 3) * 8;
          if (qq & 1) { w0 = w1; w1 = w2; w2 = w3; w3 = w4; w4 = w5; }
          if (qq & 2) { w0 = w2; w1 = w3; w2 = w4; }
          s0 = __funnelshift_r(w0, w1, bits); s1 = __funnelshift_r(w1, w2, bits);
        }
        uint8_t* rec = run.rec + static_cast<size_t>(idx) * S;
#pragma unroll
        for (int w = 0; w < NVI; w++) {
          if (w < key_vecs) {
            const uint4 m = low_bytes_mask16(static_cast<int>(ulen) - 16 * w);
            reinterpret_cast<uint4*>(rec)[w] = make_uint4(kv[w].x & m.x, kv[w].y & m.y, kv[w].z & m.z, kv[w].w & m.w);
          }
        }
        const uint8_t vfirst = vlen ? blk[p] : 0;
        uint4 tr;
        tr.x = s0; tr.y = s1;
        tr.z = ulen | (static_cast<uint32_t>(vfirst) << 16);
        tr.w = vlen;
        *reinterpret_cast<uint4*>(rec + S - 16) = tr;
        run.val_off[idx] = boff + p;
        p += vlen;
        idx++;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// K2: partition. Sample s of run r is record s*M of that run; its splitter is the row-group prefix
// of that record. pos[s_global * k + r2] = lower bound of the splitter in run r2.
struct PartView {
  const RunView* runs;          // device array [k]
  const uint32_t* sample_base;  // [k+1] prefix of samples per run
  uint32_t* pos;                // [n_samples * k]
  unsigned long long* bucket_min;   // [n_buckets]  (rank << 28 | sample)
  uint8_t* smode;               // [n_samples] 1 = the sample splits INSIDE its row group (full-key splitter)
  uint32_t n_samples;
  uint32_t n_buckets;
};

// Splitters. A sample normally stands for the START of its row group (prefix splitter), so that tiles hold whole
// groups and their retention state is self-contained. A group with more than M records in one run would pin all
// its samples to the same position and overflow a tile; such samples — recognised locally: the previous sample of
// the same run lies in the same group — split INSIDE the group at their own internal key instead (full-key
// splitter). Tiles that start there rebuild Feed's state by replaying the ancestors of their first key
// (dev_logic.cuh replay_ancestors). Candidates of one run are then < 2M records apart in that run, which bounds
// a tile by H + 2kM records (the host halves M and repeats the partition in the rare case that exceeds a tile).
constexpr unsigned long long TILE_CONT = 1ull << 63;   // tile_rank flag: the tile starts inside a row group
// Two passes: every SAMPLE_COARSE-th sample of a run searches the whole of every run (pass 0); the samples between two
// coarse ones then search only between the positions those found (pass 1) — positions are monotone in the sample index
// of a run, whichever of the two splitter kinds neighbouring samples use: ~10 probes instead of ~24, and the probes of
// neighbouring threads stay close together.
constexpr uint32_t SAMPLE_COARSE = 32;
__global__ void __launch_bounds__(256) k_sample_pos(PartView P, const JobParams* prm, JobDev* J, int pass) {
  const int S = prm->S, k = prm->k;
  const uint64_t total = static_cast<uint64_t>(P.n_samples) * k;
  for (uint64_t t = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; t < total;
       t += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const uint32_t s = static_cast<uint32_t>(t / k), r2 = static_cast<uint32_t>(t % k);
    // which run owns sample s
    int r = 0;
    while (r + 1 < k && P.sample_base[r + 1] <= s) r++;
    const uint32_t s_local = s - P.sample_base[r];
    if (((s_local % SAMPLE_COARSE) == 0) != (pass == 0)) continue;
    const uint32_t idx = s_local * prm->M;
    const uint8_t* srec = P.runs[r].rec + static_cast<size_t>(idx) * S;
    const int g = group_prefix_len(srec, rec_ulen(srec, S), prm->R.enabled != 0);
    if (g < 0) { dev_fail(J, -g, s); continue; }
    bool inside = false;
    if (idx >= prm->M) {
      const uint8_t* prec = srec - static_cast<size_t>(prm->M) * S;
      inside = rec_ulen(prec, S) >= static_cast<uint32_t>(g) && common_prefix_len(srec, g, prec, g) >= static_cast<uint32_t>(g) &&
               group_prefix_len(prec, rec_ulen(prec, S), prm->R.enabled != 0) == g;
    }
    if (r2 == 0) P.smode[s] = inside ? 1 : 0;
    const RunView& q = P.runs[r2];
    uint32_t lo = 0, hi = q.n_entries;
    if (pass == 1) {
      const uint32_t c0 = s_local - s_local % SAMPLE_COARSE, c1 = c0 + SAMPLE_COARSE;
      lo = P.pos[static_cast<size_t>(P.sample_base[r] + c0) * k + r2];
      if (P.sample_base[r] + c1 < P.sample_base[r + 1]) hi = P.pos[static_cast<size_t>(P.sample_base[r] + c1) * k + r2];
    }
    if (inside) {
      if (r2 == static_cast<uint32_t>(r)) lo = hi = idx;
      while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        const int c = cmp_records(q.rec + static_cast<size_t>(mid) * S, srec, S);
        // merged order breaks ties by run index: equal records of lower runs come first
        if (r2 < static_cast<uint32_t>(r) ? c <= 0 : c < 0) lo = mid + 1; else hi = mid;
      }
    } else {
      while (lo < hi) {
        uint32_t mid = (lo + hi) >> 1;
        const uint8_t* c = q.rec + static_cast<size_t>(mid) * S;
        // first record whose user key >= prefix
        if (cmp_prefix_vs_key(srec, g, c, rec_ulen(c, S)) > 0) lo = mid + 1; else hi = mid;
      }
    }
    P.pos[static_cast<size_t>(s) * k + r2] = lo;
  }
}

__global__ void __launch_bounds__(256) k_sample_bucket(PartView P, const JobParams* prm) {
  const int k = prm->k;
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < P.n_samples; s += gridDim.x * blockDim.x) {
    unsigned long long rank = 0;
    for (int r = 0; r < k; r++) rank += P.pos[static_cast<size_t>(s) * k + r];
    if (rank == 0) continue;                       // implicit first boundary
    uint32_t b = static_cast<uint32_t>(rank / prm->H);
    atomicMin(&P.bucket_min[b], (rank << 28) | s);
  }
}

__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* warp_sums, uint32_t* total) {
  // scan of one value per thread; all threads must call. Returns exclusive prefix.
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t x = v;
  for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  __syncthreads();
  if (lane == 31) warp_sums[wid] = x;
  __syncthreads();
  if (wid == 0) {
    uint32_t w = lane < (blockDim.x >> 5) ? warp_sums[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
    warp_sums[lane] = w;
  }
  __syncthreads();
  uint32_t excl = (wid ? warp_sums[wid - 1] : 0) + x - v;
  if (total) *total = warp_sums[(blockDim.x >> 5) - 1];
  return excl;
}

// Compact non-empty buckets into the tile boundary list. tile_lo[t*k + r] = start of tile t in
// run r; tile t ends where tile t+1 starts (last: run ends). Chunked: counts per chunk, a scan of
// the chunk counts (k_scan_u32_single), then every chunk places its tiles.
constexpr int TILE_CHUNK = 2048;
__global__ void __launch_bounds__(256) k_bucket_counts(PartView P, uint32_t* partial) {
  __shared__ uint32_t sh;
  if (threadIdx.x == 0) sh = 0;
  __syncthreads();
  const uint64_t base = static_cast<uint64_t>(blockIdx.x) * TILE_CHUNK;
  uint32_t c = 0;
  for (uint32_t j = threadIdx.x; j < TILE_CHUNK; j += 256) { const uint64_t i = base + j; if (i < P.n_buckets && P.bucket_min[i] != ~0ull) c++; }
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(&sh, c);
  __syncthreads();
  if (threadIdx.x == 0) partial[blockIdx.x] = sh;
}
__global__ void __launch_bounds__(256) k_build_tiles(PartView P, const JobParams* prm, const uint32_t* partial /*exclusive*/, const uint32_t* total,
                                                     uint32_t* tile_lo, unsigned long long* tile_rank, JobDev* J) {
  __shared__ uint32_t warp_sums[32];
  const int k = prm->k;
  if (blockIdx.x == 0) {                           // tile 0 = implicit boundary at all-zero
    if (threadIdx.x < k) tile_lo[threadIdx.x] = 0;
    if (threadIdx.x == 0) { tile_rank[0] = 0; J->n_tiles = *total + 1; }
  }
  const uint64_t base = static_cast<uint64_t>(blockIdx.x) * TILE_CHUNK;
  constexpr int PER = TILE_CHUNK / 256;
  unsigned long long v[PER];
  uint32_t c = 0;
  for (int j = 0; j < PER; j++) { const uint64_t i = base + threadIdx.x * PER + j; v[j] = i < P.n_buckets ? P.bucket_min[i] : ~0ull; c += v[j] != ~0ull; }
  uint32_t t = 1 + partial[blockIdx.x] + block_exclusive_scan(c, warp_sums, nullptr);
  for (int j = 0; j < PER; j++) {
    if (v[j] == ~0ull) continue;
    const uint32_t s = static_cast<uint32_t>(v[j] & ((1u << 28) - 1));
    for (int r = 0; r < k; r++) tile_lo[static_cast<size_t>(t) * k + r] = P.pos[static_cast<size_t>(s) * k + r];
    tile_rank[t] = (v[j] >> 28) | (P.smode[s] ? TILE_CONT : 0ull);
    t++;
  }
}

// Largest tile of the partition (the host repeats the partition with a smaller sample stride if it exceeds a tile).
__global__ void __launch_bounds__(256) k_tile_check(const RunView* runs, const uint32_t* tile_lo, int k, JobDev* J) {
  const uint32_t n_tiles = J->n_tiles;
  uint32_t mx = 0;
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n_tiles; t += gridDim.x * blockDim.x) {
    uint32_t sz = 0;
    for (int r = 0; r < k; r++) {
      const uint32_t lo = tile_lo[static_cast<size_t>(t) * k + r];
      const uint32_t hi = (t + 1 < n_tiles) ? tile_lo[static_cast<size_t>(t + 1) * k + r] : runs[r].n_entries;
      sz += hi - lo;
    }
    mx = max(mx, sz);
  }
  mx = __reduce_max_sync(0xffffffffu, mx);
  if ((threadIdx.x & 31) == 0 && mx) atomicMax(&J->max_tile, mx);
}

// ---------------------------------------------------------------------------------------------
// K3: merge + filter, one CTA per tile.
struct MergeView {
  const RunView* runs;            // [k]
  const uint32_t* tile_lo;        // [n_tiles * k]
  const unsigned long long* tile_rank;   // [n_tiles] rank (merged position) of the tile's first entry
  Desc* desc;                     // [N]
  ValueRewrite* rewrites;         // [rewrite_cap]
  uint32_t rewrite_cap;
  uint32_t n_tiles;
  uint16_t* fk16;                 // [N] by input entry id: bloom filter key length (nullptr = no filter policy)
  uint32_t* fkh;                  // [N] by input entry id: bloom hash of that filter key (the record is in shared memory here;
                                  //     the filter builder would have to gather it from HBM again); nullptr = not wanted
  int32_t S, k;                   // record stride / number of runs / tile capacity: kernel-parameter constants
  uint32_t cap;
};

constexpr int MERGE_THREADS = 256;
constexpr uint8_t ENT_GROUP_START = 128;           // tile-local: first entry of a row group (never leaves the merge kernel)
constexpr uint32_t RW_PRE_DROPPED = 0xfffffffeu;   // rw_slot marker: dropped as an overwritten older version
constexpr int RANK_C = 8;        // coarse stride of the two-level rank search
constexpr int RANK_KMAX = 16;    // two-level search used for k <= RANK_KMAX runs

// Shared-memory layout of a merge tile. Every array base is FIXED + cap * K with compile-time FIXED
// and K (cap is a multiple of 16, so all alignments hold by construction): a base costs one
// multiply-add wherever it is needed instead of a chain of dependent pointer computations.
namespace tile_layout {
constexpr uint32_t SEG_LO = 0;                                  // u32 [MAX_RUNS]
constexpr uint32_t SEG_START = SEG_LO + 4 * MAX_RUNS;           // u32 [MAX_RUNS + 1]
constexpr uint32_t CBASE = SEG_START + 4 * (MAX_RUNS + 2);      // u32 [MAX_RUNS + 1] coarse index base per segment
constexpr uint32_t CRANK = CBASE + 4 * (MAX_RUNS + 2);          // u16 [(cap / RANK_C + RANK_KMAX + 1) * RANK_KMAX] coarse ranks
constexpr uint32_t CRANK_FIXED = 2 * (RANK_KMAX + 1) * RANK_KMAX;
constexpr uint32_t CRANK_PER = 2 * RANK_KMAX / RANK_C;          // bytes per record
constexpr uint32_t A0 = (CRANK + CRANK_FIXED + 15) & ~15u;
constexpr uint32_t ORDER_K = CRANK_PER;      // u16 sorted pos -> local idx
constexpr uint32_t GLEN_K = ORDER_K + 2;     // u16 local idx -> group prefix len
constexpr uint32_t GSTART_K = GLEN_K + 2;    // u16 group -> first sorted pos (cap + 2 entries; +16 bytes below)
constexpr uint32_t A1 = A0 + 16;
constexpr uint32_t PVIS_K = GSTART_K + 2;    // u16 sorted pos -> previous visible sorted pos
constexpr uint32_t RES_K = PVIS_K + 2;       // u8 sorted pos -> ENT_* flags
constexpr uint32_t RW_K = RES_K + 1;         // u32 sorted pos -> rewrite slot
constexpr uint32_t PFX_K = RW_K + 4;         // u64 local idx -> sort prefix
constexpr uint32_t PFX2_K = PFX_K + 8;       // u64 second 8 bytes of the 16-byte sort prefix
constexpr uint32_t RECS_K = PFX2_K + 8;      // records, SS bytes each
static_assert(RANK_KMAX % RANK_C == 0 && (PFX_K % 1) == 0, "layout");
__host__ __device__ constexpr uint32_t bytes(uint32_t S, uint32_t cap) { return A1 + (RECS_K + S + 8) * cap; }
}  // namespace tile_layout

// A staged record's 8 bytes of bank padding (stride S + 8) hold its run and its index in that run, written by the
// staging loop that already knows both: no later pass searches the segment bounds for them.
__device__ __forceinline__ uint32_t staged_run(const uint8_t* rec, int S) { return *reinterpret_cast<const uint32_t*>(rec + S); }
__device__ __forceinline__ uint32_t staged_idx(const uint8_t* rec, int S) { return *reinterpret_cast<const uint32_t*>(rec + S + 4); }


static_assert(MAX_RUNS <= REPLAY_MAX_RUNS, "a replay's cursors cover every run of a job");

// One thread, rare: the run table for replay_ancestors lives in this function's frame, not in the kernel's.
__device__ __noinline__ int seed_continuation(FeedState* st, const JobParams* prm, const RunView* runs, const uint32_t* seg_lo, int k, int S,
                                              const uint8_t* k0_smem) {
  ReplayRun rr[REPLAY_MAX_RUNS];
  for (int r = 0; r < k; r++) { rr[r].rec = runs[r].rec; rr[r].limit = seg_lo[r]; rr[r].data = runs[r].data; rr[r].val_off = runs[r].val_off; }
  return replay_ancestors(st, prm->R, rr, k, S, k0_smem, rec_ulen(k0_smem, S), prm->bottommost, prm->last_sequence);
}

// Id length of a cotable ('y') / colocated ('0') key, 0 for any other key (the key was validated by group_prefix_len).
__device__ __forceinline__ int table_id_len(const uint8_t* e, uint32_t ulen) {
  return (e[0] == 'y' || e[0] == '0') ? dockey_id_size(e, ulen) : 0;
}

// The one table of a tile whose tombstones may lie outside it: the table of the tile's first record. One thread, at
// most once per tile: slot 0 of that table's rows from its tombstones in the runs — below the tile, or up to the tile's
// end when the tile starts inside the tombstone group (`through_tile`). Returns 1 when the rows start from the
// table-level overwrite *ow0, 0 when they start fresh, or a negative DevError.
__device__ __noinline__ int seed_table_from_runs(Overwrite* ow0, const JobParams* prm, const RunView* runs, const uint32_t* seg_lo,
                                                 const uint32_t* seg_start, int k, int S, const uint8_t* row, int id, bool through_tile) {
  ReplayRun rr[REPLAY_MAX_RUNS];
  for (int r = 0; r < k; r++) {
    rr[r].rec = runs[r].rec; rr[r].data = runs[r].data; rr[r].val_off = runs[r].val_off;
    rr[r].limit = seg_lo[r] + (through_tile ? seg_start[r + 1] - seg_start[r] : 0u);
  }
  FeedState st;
  const int d = replay_table_seed(&st, prm->R, rr, k, S, row, static_cast<uint32_t>(id), prm->bottommost, prm->last_sequence);
  if (d < 0) return d;
  if (!st.n_ow) return 0;
  *ow0 = st.ow[0];
  return 1;
}

// Every other table of the tile: its tombstone group, sorted positions [i0, i1), is in shared memory. A row group of the
// table replays it on *st (fresh) and turns the result into its starting state (table_seed).
__device__ __noinline__ int seed_table_in_tile(FeedState* st, const JobParams* prm, const RunView* runs, const uint8_t* recs, int SS, int S,
                                               const uint16_t* order, uint32_t i0, uint32_t i1, const uint8_t* row, int id) {
  feed_state_reset(st);
  const uint8_t* prev = nullptr;
  for (uint32_t i = i0; i < i1; i++) {
    const uint8_t* c = recs + static_cast<size_t>(SS) * order[i];
    if (rec_flags(c, S) & REC_F_HT_FILTERED) continue;           // out-of-range tombstones DO seed the table state
    const uint8_t* val = nullptr;
    if (rec_vlen(c, S) && has_control_fields(rec_vfirst(c, S))) {
      const uint32_t r = staged_run(c, S);
      val = runs[r].data + runs[r].val_off[staged_idx(c, S)];
    }
    const int d = replay_entry(st, prm->R, c, S, val, &prev, prm->bottommost, prm->last_sequence);
    if (d < 0) return d;
  }
  table_seed(st, row, static_cast<uint32_t>(id));
  return 0;
}

// Fast path of the retention pass: every visible entry of the row group, sorted positions [i0, i1), is newer than the
// history cutoff and is a plain value of an ordinary table key. Feed forwards such entries verbatim
// (docdb_compaction_context.cc:1117-1130) and the row's overwrite stack is never consulted, so the state machine can be
// skipped (subkey decoding errors of such rows are not diagnosed).
__device__ __forceinline__ bool row_above_cutoff(const JobParams* prm, const uint8_t* recs, int SS, int S, const uint16_t* order,
                                                 const uint8_t* res, uint32_t i0, uint32_t i1) {
  if (prm->R.lower_len | prm->R.upper_len) return false;
  for (uint32_t i = i0; i < i1; i++) {
    if (!(res[i] & ENT_KEEP)) continue;
    const uint8_t* e = recs + static_cast<size_t>(SS) * (order[i]);
    const uint32_t ulen = rec_ulen(e, S);
    const uint8_t b0 = ulen ? e[0] : 10;
    const uint32_t htl = doc_ht_len_from_end(e, ulen);
    const uint8_t vf = rec_vfirst(e, S);
    if (b0 == 10 || b0 == 6 || b0 == 7 || b0 == 'y' || b0 == '0' || !htl ||
        encht_cmp(e + ulen - htl, htl, prm->R.cutoff_enc.b, prm->R.cutoff_enc.n) <= 0 ||
        (rec_vlen(e, S) && (has_control_fields(vf) || vf == 'z' || vf == '|')))
      return false;
  }
  return true;
}

// Row group g, sorted positions [gstart[g], gstart[g + 1]), through DocDBCompactionFeed::Feed (feed_step), serially by
// one thread. Its FeedState lives in this function's frame, not in the kernel's: only groups the fast path does not
// cover pay for it. `id` > 0: the group is a row of a cotable / colocated table with that id length, seeded from its
// table's tombstones (blk[g] = the first group of its id block). `continued`: the group began in an earlier tile.
// Returns the number of entries Feed dropped.
__device__ __noinline__ uint32_t feed_row(const JobParams* prm, JobDev* J, const RunView* runs, ValueRewrite* rewrites, uint32_t rewrite_cap,
                                          const uint32_t* seg_lo, int k, const uint8_t* recs, int SS, int S, const uint16_t* order,
                                          const uint16_t* gstart, const uint16_t* blk, uint8_t* res, uint32_t* rw_slot, uint32_t g, int id,
                                          bool continued, int ow0_state, const Overwrite* ow0, uint32_t tile) {
  FeedState st;
  feed_state_reset(&st);
  const uint32_t i0 = gstart[g], i1 = gstart[g + 1];
  if (id > 0) {
    const uint8_t* e0 = recs + static_cast<size_t>(SS) * order[i0];
    const uint32_t h = blk[g];
    if (h == 0 && ow0_state) {
      if (ow0_state == 2) feed_state_seed(&st, e0, id, *ow0);
    } else if (recs[static_cast<size_t>(SS) * order[gstart[h]] + id] == '!') {   // the block starts with the tombstones
      const int rc = seed_table_in_tile(&st, prm, runs, recs, SS, S, order, gstart[h], gstart[h + 1], e0, id);
      if (rc < 0) { dev_fail(J, -rc, tile); return 0; }
    }
  }
  if (continued) {
    // Rebuild Feed's state at the tile's first record from the entries that determine it (its ancestors `P_i # HT`
    // and the earlier versions of its own SubDocKey).
    const int rc = seed_continuation(&st, prm, runs, seg_lo, k, S, recs + static_cast<size_t>(SS) * order[i0]);
    if (rc < 0) { dev_fail(J, -rc, tile); return 0; }
  }
  uint32_t dropped = 0;
  for (uint32_t i = i0; i < i1; i++) {
    uint8_t f = res[i];
    if (!(f & ENT_KEEP)) continue;
    if (rw_slot[i] == RW_PRE_DROPPED) { rw_slot[i] = 0xffffffffu; res[i] = f & ~ENT_KEEP & ~ENT_ZERO_SEQ; dropped++; continue; }
    const uint8_t* e = recs + static_cast<size_t>(SS) * order[i];
    const uint32_t vlen = rec_vlen(e, S);
    const uint8_t vfirst = rec_vfirst(e, S);
    const uint8_t* val = nullptr;
    if (vlen && has_control_fields(vfirst)) { const uint32_t r = staged_run(e, S); val = runs[r].data + runs[r].val_off[staged_idx(e, S)]; }
    ValueRewrite rw;
    int d = feed_step(&st, prm->R, e, rec_ulen(e, S), vfirst, val, vlen, &rw);
    if (d < 0) { dev_fail(J, -d, tile); break; }
    if (d == 0) { res[i] = f & ~ENT_KEEP & ~ENT_ZERO_SEQ; dropped++; continue; }
    f |= static_cast<uint8_t>(d);
    if (d & ENT_VAL_REENCODE) {
      uint32_t slot = atomicAdd(&J->n_rewrites, 1u);
      if (slot < rewrite_cap) { rewrites[slot] = rw; rw_slot[i] = slot; }
      else dev_fail(J, DEV_ERR_UNSUPPORTED_VALUE, tile);
    }
    res[i] = f;
  }
  return dropped;
}

// 8-byte asynchronous copy global -> shared (the 16-byte form needs a 16-byte aligned destination), and the wait for
// all of a thread's copies.
__device__ __forceinline__ void cp_async_8(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(dst))), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// Exclusive max-scan of one value per thread (0 for thread 0); all threads must call.
__device__ __forceinline__ uint32_t block_exclusive_max(uint32_t v, uint32_t* warp_sums) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t x = v;
  for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x = max(x, y); }
  uint32_t ex = __shfl_up_sync(0xffffffffu, x, 1);
  if (lane == 0) ex = 0;
  __syncthreads();
  if (lane == 31) warp_sums[wid] = x;
  __syncthreads();
  if (wid == 0) {
    uint32_t m = lane < (blockDim.x >> 5) ? warp_sums[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, m, o); if (lane >= o) m = max(m, y); }
    warp_sums[lane] = m;
  }
  __syncthreads();
  return max(wid ? warp_sums[wid - 1] : 0u, ex);
}

__global__ void __launch_bounds__(MERGE_THREADS, 3) k_merge_filter(MergeView V, const JobParams* prm, JobDev* J) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int S = V.S, k = V.k;
  const int SS = S + 8;                       // smem record stride: +8 B so that consecutive records start in different banks
  const uint32_t cap = V.cap;
  namespace L = tile_layout;
  uint32_t* seg_lo = reinterpret_cast<uint32_t*>(smem + L::SEG_LO);
  uint32_t* seg_start = reinterpret_cast<uint32_t*>(smem + L::SEG_START);
  uint32_t* cbase = reinterpret_cast<uint32_t*>(smem + L::CBASE);
  uint16_t* crank = reinterpret_cast<uint16_t*>(smem + L::CRANK);
  uint16_t* order = reinterpret_cast<uint16_t*>(smem + L::A0 + L::ORDER_K * cap);
  uint16_t* glen = reinterpret_cast<uint16_t*>(smem + L::A0 + L::GLEN_K * cap);
  uint16_t* gstart = reinterpret_cast<uint16_t*>(smem + L::A0 + L::GSTART_K * cap);
  uint16_t* pvis = reinterpret_cast<uint16_t*>(smem + L::A1 + L::PVIS_K * cap);
  uint8_t* res = smem + L::A1 + L::RES_K * cap;
  uint32_t* rw_slot = reinterpret_cast<uint32_t*>(smem + L::A1 + L::RW_K * cap);
  unsigned long long* pfx = reinterpret_cast<unsigned long long*>(smem + L::A1 + L::PFX_K * cap);
  unsigned long long* pfx2 = reinterpret_cast<unsigned long long*>(smem + L::A1 + L::PFX2_K * cap);
  uint8_t* recs = smem + L::A1 + L::RECS_K * cap;                   // cap * SS
  __shared__ uint32_t warp_sums[32];
  __shared__ uint32_t sh_T, sh_ngroups, sh_any_filtered, sh_any_id;
  __shared__ int sh_err;
  __shared__ uint32_t sh_c0;
  __shared__ Overwrite sh_ow0;                   // slot 0 for the rows of the table the tile starts in, when looked up in the runs
  __shared__ int sh_ow0_state;                   // 0 = not looked up, 1 = the rows start fresh, 2 = they start from sh_ow0
  __shared__ const uint8_t* sh_pred;             // tile that starts inside a row group: the last visible record before it
  __shared__ uint32_t sh_rb[2][MAX_RUNS + 2];    // run boundaries of the merge tree (ping-pong per level)

  const uint32_t tile = blockIdx.x;
  const bool cont = (V.tile_rank[tile] & TILE_CONT) != 0;
  if (threadIdx.x < 32) {
    // segment bounds: one lane per run (k <= MAX_RUNS), prefix sum by shuffles; the job's error word rides along so
    // that no thread has to fetch it from HBM in the middle of the tile
    static_assert(MAX_RUNS <= 64, "two rounds of 32 lanes cover the runs");
    uint32_t acc = 0;
    for (int r0 = 0; r0 < k; r0 += 32) {
      const int r = r0 + static_cast<int>(threadIdx.x);
      uint32_t lo = 0, n = 0;
      if (r < k) {
        lo = V.tile_lo[static_cast<size_t>(tile) * k + r];
        const uint32_t hi = (tile + 1 < V.n_tiles) ? V.tile_lo[static_cast<size_t>(tile + 1) * k + r] : V.runs[r].n_entries;
        n = hi - lo;
      }
      uint32_t x = n;
      for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (static_cast<int>(threadIdx.x) >= o) x += y; }
      if (r < k) { seg_lo[r] = lo; seg_start[r] = acc + x - n; }
      acc += __shfl_sync(0xffffffffu, x, 31);
    }
    if (threadIdx.x == 0) {
      seg_start[k] = acc;
      sh_T = acc;
      sh_any_filtered = 0;
      sh_any_id = 0;
      sh_err = *reinterpret_cast<volatile int*>(&J->error);
    }
  }
  __syncthreads();
  const uint32_t T = sh_T;
  if (T == 0) return;
  if (cont && threadIdx.x == 0) atomicAdd(&J->n_cont_tiles, 1u);
  if (T > cap) { if (threadIdx.x == 0) dev_fail(J, DEV_ERR_TILE_OVERFLOW, tile); return; }

  // (a) stage the k segments from HBM, re-strided to SS in smem: ONE flat loop over all the tile's 16-byte vectors, each
  // copied by two asynchronous 8-byte copies (SS is only 8-byte aligned). No load result passes through a register, so
  // all of a thread's ~15 copies are in flight together and the tile waits for HBM once; register loads waited once per
  // vector, because the run search between them kept the compiler from batching them.
  {
    const uint32_t vpr = S >> 4;                      // 16-byte vectors per record
    const uint32_t nvec = T * vpr;
    const bool vpr_pow2 = (vpr & (vpr - 1)) == 0;
    const uint32_t vpr_shift = 31 - __clz(vpr);
    int r = 0;                                        // a thread's records only move forward: so does its run
#pragma unroll 4
    for (uint32_t i = threadIdx.x; i < nvec; i += blockDim.x) {
      const uint32_t li = vpr_pow2 ? i >> vpr_shift : i / vpr, q = i - li * vpr;
      while (seg_start[r + 1] <= li) r++;
      const uint32_t idx = seg_lo[r] + (li - seg_start[r]);
      const uint8_t* src = V.runs[r].rec + static_cast<size_t>(idx) * S + 16 * q;
      uint8_t* dst = recs + static_cast<size_t>(li) * SS + 16 * q;
      cp_async_8(dst, src);
      cp_async_8(dst + 8, src + 8);
      if (q == 0) *reinterpret_cast<uint2*>(recs + static_cast<size_t>(li) * SS + S) = make_uint2(static_cast<uint32_t>(r), idx);
    }
    cp_async_wait_all();
  }
  __syncthreads();

  // tile-common key prefix -> 8-byte sort prefixes (most comparisons are decided by one u64)
  if (threadIdx.x < 32) {
    // The prefix common to every key of the tile = min over the segments' first and last keys of their common prefix
    // with any one key of the tile (the segments are sorted): one lane per segment instead of a serial min / max search
    // by one thread while the CTA waits.
    const uint8_t* ref = recs;                         // local record 0 (T > 0)
    const uint32_t ref_len = rec_ulen(ref, S);
    uint32_t c = 0xffffffffu;
    for (int r = static_cast<int>(threadIdx.x); r < k; r += 32) {
      const uint32_t n = seg_start[r + 1] - seg_start[r];
      if (!n) continue;
      const uint8_t* f = recs + static_cast<size_t>(SS) * seg_start[r];
      const uint8_t* l = recs + static_cast<size_t>(SS) * (seg_start[r + 1] - 1);
      c = min(c, min(common_prefix_len(ref, ref_len, f, rec_ulen(f, S)), common_prefix_len(ref, ref_len, l, rec_ulen(l, S))));
    }
    c = __reduce_min_sync(0xffffffffu, c);
    c = min(c, ref_len) & ~7u;
    if (c + 16 > static_cast<uint32_t>(S - 16)) c = (S - 16 >= 16) ? static_cast<uint32_t>(S - 32) & ~7u : 0;
    if (threadIdx.x == 0) sh_c0 = c;
  }
  if (threadIdx.x == 0) {
    // A tile that starts inside a row group needs the record that precedes it in merged order (rule A compares
    // with the previous visible user key): the largest visible record below the tile's start over all runs.
    const uint8_t* pred = nullptr;
    if (cont) {
      for (int r = 0; r < k; r++) {
        uint32_t j = seg_lo[r];
        const uint8_t* c2 = nullptr;
        while (j > 0) {
          const uint8_t* q = V.runs[r].rec + static_cast<size_t>(j - 1) * S;
          if (!(rec_flags(q, S) & REC_F_INVISIBLE)) { c2 = q; break; }
          j--;
        }
        if (c2 && (!pred || cmp_records(c2, pred, S) >= 0)) pred = c2;     // ties: the higher run comes later
      }
    }
    sh_pred = pred;
  }
  __syncthreads();
  {
    const uint32_t c0 = sh_c0;
    for (uint32_t li = threadIdx.x; li < T; li += blockDim.x)
    {
      pfx[li] = bswap64(ld_u64_aligned(recs + static_cast<size_t>(SS) * li + c0));
      pfx2[li] = bswap64(ld_u64_aligned(recs + static_cast<size_t>(SS) * li + c0 + 8));
    }
  }
  __syncthreads();

  // (b) k-way merge of the sorted segments: a binary tree of pairwise merges in shared memory. On every level
  // each thread produces MT consecutive output positions of one pair of neighbouring runs: a merge-path search
  // along its diagonal finds where the two runs are cut, then MT sequential merge steps follow. Only the u16
  // permutation moves (ping-pong between `order` and the former coarse-rank area); comparisons go through the
  // 16-byte sort prefixes and fall back to the full record compare on ties. Records of the lower-numbered run
  // come first among equals (the order the reference's MergingIterator heap produces for equal internal keys is
  // never observable: sequence numbers are unique across files — table/merger.cc:652-697).
  // ~log2(k) x (log2(n) probes + MT steps) per MT records instead of (k - 1) binary searches per record.
  {
    constexpr int MT = 2;
    uint16_t* bufs[2] = {order, reinterpret_cast<uint16_t*>(crank)};
    // a <= b in merged order, a from the earlier run group
    auto le = [&](uint32_t a, uint32_t b) -> bool {
      const unsigned long long pa = pfx[a], pb = pfx[b];
      if (pa != pb) return pa < pb;
      const unsigned long long qa = pfx2[a], qb = pfx2[b];
      if (qa != qb) return qa < qb;
      return cmp_records(recs + static_cast<size_t>(SS) * a, recs + static_cast<size_t>(SS) * b, S) <= 0;
    };
    for (uint32_t li = threadIdx.x; li < T; li += blockDim.x) bufs[0][li] = static_cast<uint16_t>(li);
    if (threadIdx.x <= static_cast<uint32_t>(k)) sh_rb[0][threadIdx.x] = seg_start[threadIdx.x];
    __syncthreads();
    int nruns = k, cur = 0;
    while (nruns > 1) {
      const uint16_t* src = bufs[cur]; uint16_t* dst = bufs[cur ^ 1];
      const uint32_t* rb = sh_rb[cur];
      const int npairs = (nruns + 1) >> 1;
      for (uint32_t o0 = threadIdx.x * MT; o0 < T; o0 += blockDim.x * MT) {
        int p = 0;
        while (p + 1 < npairs && rb[2 * (p + 1)] <= o0) p++;
        uint32_t a0 = rb[2 * p], a1 = rb[min(2 * p + 1, nruns)], b1 = rb[min(2 * p + 2, nruns)];
        // merge path: how many of the first d outputs of this pair come from A = src[a0, a1) (B = src[a1, b1))
        const uint32_t d = o0 - a0, la = a1 - a0, lb = b1 - a1;
        uint32_t lo = d > lb ? d - lb : 0, hi = min(d, la);
        while (lo < hi) {
          const uint32_t mid = (lo + hi) >> 1;
          if (le(src[a0 + mid], src[a1 + (d - 1 - mid)])) lo = mid + 1; else hi = mid;
        }
        uint32_t i = a0 + lo, j = a1 + (d - lo);
        const uint32_t o_end = min(o0 + MT, T);
        for (uint32_t o = o0; o < o_end; o++) {
          while (o == b1 && p + 1 < npairs) {              // the chunk runs into the next (non-empty) pair
            p++;
            a0 = rb[2 * p]; a1 = rb[min(2 * p + 1, nruns)]; b1 = rb[min(2 * p + 2, nruns)];
            i = a0; j = a1;
          }
          uint16_t pick;
          if (i < a1 && (j >= b1 || le(src[i], src[j]))) pick = src[i++]; else pick = src[j++];
          dst[o] = pick;
        }
      }
      if (threadIdx.x <= static_cast<uint32_t>(npairs)) sh_rb[cur ^ 1][threadIdx.x] = rb[min(2 * static_cast<int>(threadIdx.x), nruns)];
      __syncthreads();
      nruns = npairs; cur ^= 1;
    }
    if (cur) {                                             // the permutation must end up in `order`
      for (uint32_t li = threadIdx.x; li < T; li += blockDim.x) order[li] = bufs[1][li];
    }
  }
  // per record: input order check, row-group prefix, bloom filter key length
  for (uint32_t li = threadIdx.x; li < T; li += blockDim.x) {
    const uint8_t* e = recs + static_cast<size_t>(SS) * li;
    const uint32_t r = staged_run(e, S);
    if (li > seg_start[r] && cmp_records(e - SS, e, S) >= 0) { dev_fail(J, DEV_ERR_UNSORTED, tile); sh_err = 1; }
    int fk = 0;
    const int g = group_prefix_len(e, rec_ulen(e, S), prm->R.enabled != 0, V.fk16 ? &fk : nullptr);
    if (g < 0) { dev_fail(J, -g, tile); sh_err = 1; glen[li] = 0; } else glen[li] = static_cast<uint16_t>(g);
    if (V.fk16) {
      const uint32_t gid = V.runs[r].gid_base + staged_idx(e, S);
      V.fk16[gid] = static_cast<uint16_t>(g < 0 ? 0 : fk);
      if (V.fkh) V.fkh[gid] = (g < 0 || fk <= 0) ? 0u : leveldb_hash(e, static_cast<uint32_t>(fk), kBloomSeed);
    }
    if (rec_flags(e, S) & REC_F_INVISIBLE) sh_any_filtered = 1;
    if (e[0] == 'y' || e[0] == '0') sh_any_id = 1;
  }
  __syncthreads();
  if (sh_err) return;                              // the job had failed already, or this tile's records are bad

  // previous-visible map (identity - 1 unless HybridTime-filtered entries exist)
  if (sh_any_filtered) {
    if (threadIdx.x == 0) {
      uint32_t last = 0xffff;
      for (uint32_t i = 0; i < T; i++) {
        pvis[i] = static_cast<uint16_t>(last);
        if (!(rec_flags(recs + static_cast<size_t>(SS) * (order[i]), S) & REC_F_INVISIBLE)) last = i;
      }
    }
  } else {
    for (uint32_t i = threadIdx.x; i < T; i += blockDim.x) pvis[i] = static_cast<uint16_t>(i ? i - 1 : 0xffff);
  }
  __syncthreads();

  // (c) CompactionIterator per sorted position + group starts
  const uint32_t items = (T + blockDim.x - 1) / blockDim.x;          // consecutive items per thread
  uint32_t my_groups = 0;
  unsigned long long st_counted = 0, st_hidden = 0, st_obsolete = 0, st_in_k = 0, st_in_v = 0;
  for (uint32_t j = 0; j < items; j++) {
    const uint32_t i = threadIdx.x * items + j;
    if (i >= T) break;
    const uint32_t li = order[i];
    const uint8_t* e = recs + static_cast<size_t>(SS) * (li);
    uint8_t f = 0;
    if (!(rec_flags(e, S) & REC_F_INVISIBLE)) {
      f |= ENT_COUNTED; st_counted++;
      st_in_k += rec_ulen(e, S) + 8; st_in_v += rec_vlen(e, S);
      const uint64_t suffix = rec_suffix(e, S);
      const uint32_t type = static_cast<uint32_t>(suffix & 0xff);
      const uint64_t seq = suffix >> 8;
      if (type != 0 && type != 1) dev_fail(J, DEV_ERR_UNSUPPORTED_VALUE, tile);     // merge / single delete
      const uint32_t ulen = rec_ulen(e, S);
      bool first_occ = true;
      if (pvis[i] != 0xffff) {
        const uint8_t* pe = recs + static_cast<size_t>(SS) * (order[pvis[i]]);
        first_occ = cmp_user_keys(pe, rec_ulen(pe, S), e, ulen) != 0;
      } else if (cont && sh_pred) {
        first_occ = cmp_user_keys(sh_pred, rec_ulen(sh_pred, S), e, ulen) != 0;   // previous visible record lies in an earlier tile
      }
      if (!first_occ) { f |= ENT_DROP_HIDDEN; st_hidden++; }                       // rule A
      else if (type == 0 && prm->bottommost && seq <= prm->last_sequence) { f |= ENT_DROP_OBSOLETE; st_obsolete++; }
      else {
        f |= ENT_KEEP;
        if (prm->bottommost && seq < prm->last_sequence) {                         // PrepareOutput
          bool is_largest = ulen == prm->largest_len;
          for (uint32_t q = 0; is_largest && q < ulen; q++) is_largest = e[q] == prm->largest[q];
          if (!is_largest) f |= ENT_ZERO_SEQ;
        }
      }
    }
    bool gs = i == 0;
    if (!gs) {
      const uint32_t lp = order[i - 1];
      const uint32_t g = glen[li];
      gs = glen[lp] != g || common_prefix_len(e, g, recs + static_cast<size_t>(SS) * (lp), g) < g;
    }
    if (gs) { my_groups++; f |= ENT_GROUP_START; }
    res[i] = f;
  }
  uint32_t ngroups;
  uint32_t gbase = block_exclusive_scan(my_groups, warp_sums, &ngroups);
  for (uint32_t j = 0; j < items; j++) {
    const uint32_t i = threadIdx.x * items + j;
    if (i >= T) break;
    if (res[i] & ENT_GROUP_START) gstart[gbase++] = static_cast<uint16_t>(i);
  }
  if (threadIdx.x == 0) { gstart[ngroups] = static_cast<uint16_t>(T); sh_ngroups = ngroups; }
  __syncthreads();

  // (d) DocDB retention predicate: one thread per row group, serial inside the group
  unsigned long long st_feed = 0;
  for (uint32_t i = threadIdx.x; i < T; i += blockDim.x) {
    uint32_t mark = 0xffffffffu;
    // Older versions of one SubDocKey: when the entry fed just before this one has the same key
    // up to the hybrid time, is at or below the history cutoff and neither is a TTL merge record,
    // Feed has (at least) that entry's time on top of the overwrite stack and drops this one at
    // docdb_compaction_context.cc:1067-1074 without touching its state. Decided here by all
    // threads so that the serial walk of a row group only visits entries that can survive.
    if (i > 0 && prm->R.enabled && (res[i] & ENT_KEEP) && (res[i - 1] & ENT_KEEP)) {
      const uint8_t* e = recs + static_cast<size_t>(SS) * order[i];
      const uint8_t* p = recs + static_cast<size_t>(SS) * order[i - 1];
      const uint32_t ul = rec_ulen(e, S), pl = rec_ulen(p, S);
      const uint32_t hl = doc_ht_len_from_end(e, ul), hp = doc_ht_len_from_end(p, pl);
      if (hl && hp && ul - hl == pl - hp &&
          !(rec_vlen(e, S) && rec_vfirst(e, S) == 'k') && !(rec_vlen(p, S) && rec_vfirst(p, S) == 'k')) {
        const EncHt& chosen = (e[0] == 'y' && prm->R.has_cotables_cutoff) ? prm->R.cotables_cutoff_enc : prm->R.cutoff_enc;
        if (encht_cmp(p + pl - hp, hp, chosen.b, chosen.n) <= 0 && common_prefix_len(e, ul - hl, p, ul - hl) >= ul - hl)
          mark = RW_PRE_DROPPED;
      }
    }
    rw_slot[i] = mark;
  }
  // (d0) cotable / colocated tables: slot 0 of the overwrite stack (the table tombstones' time) carries over all rows
  // of a table. The tombstones `id ! # HT` sort before every row of their table, as one row group. The tile holds every
  // entry between two splitters, so every id block of the tile (a maximal run of row groups with one id) other than the
  // one the tile starts in also holds its table's tombstones, as its first group: a row group of such a table replays
  // that group from shared memory. Only the block the tile starts in can have its tombstones in earlier tiles: thread 0
  // replays them from the runs, once. Tiles stay independent, and tiles without 'y' / '0' keys skip all of this.
  // After the scan, pvis[g] = the first group of the id block of group g (pvis is free once (c) is done).
  const bool ids = prm->R.enabled && sh_any_id;
  if (ids) {
    const uint32_t ngroups = sh_ngroups;
    if (threadIdx.x == 0) {
      int state = 0;
      const uint8_t* e = recs + static_cast<size_t>(SS) * order[0];
      const uint32_t ul = rec_ulen(e, S);
      const int id = table_id_len(e, ul);
      if (id > 0 && static_cast<uint32_t>(id) < ul) {
        bool lookup = e[id] != '!';                     // the tile starts among the table's rows
        if (!lookup && cont && ngroups > 1) {           // it starts inside the tombstones: only rows of the table need them
          const uint8_t* n1 = recs + static_cast<size_t>(SS) * order[gstart[1]];
          lookup = rec_ulen(n1, S) > static_cast<uint32_t>(id) && n1[id] != '!' && common_prefix_len(n1, id, e, id) >= static_cast<uint32_t>(id);
        }
        if (lookup) {
          const int rc = seed_table_from_runs(&sh_ow0, prm, V.runs, seg_lo, seg_start, k, S, e, id, e[id] == '!');
          if (rc < 0) dev_fail(J, -rc, tile);
          state = rc > 0 ? 2 : 1;
        }
      }
      sh_ow0_state = state;
    }
    // mark every group that starts an id block (or has no id), then a max-scan carries the marks over the groups
    const uint32_t per = (ngroups + blockDim.x - 1) / blockDim.x;
    const uint32_t g0 = min(threadIdx.x * per, ngroups), g1 = min(g0 + per, ngroups);
    uint32_t last = 0;                                  // 1 + the last mark in this thread's groups, 0 = none yet
    for (uint32_t g = g0; g < g1; g++) {
      bool head = g == 0;
      if (!head) {
        const uint8_t* e = recs + static_cast<size_t>(SS) * order[gstart[g]];
        const uint8_t* p = recs + static_cast<size_t>(SS) * order[gstart[g - 1]];
        const int id = table_id_len(e, rec_ulen(e, S));
        head = id <= 0 || table_id_len(p, rec_ulen(p, S)) != id || common_prefix_len(p, id, e, id) < static_cast<uint32_t>(id);
      }
      if (head) last = g + 1;
      pvis[g] = static_cast<uint16_t>(last ? last - 1 : 0xffff);
    }
    const uint32_t carry = block_exclusive_max(last, warp_sums);
    for (uint32_t g = g0; g < g1 && pvis[g] == 0xffff; g++) pvis[g] = static_cast<uint16_t>(carry - 1);
  }
  __syncthreads();
  if (prm->R.enabled) {
    for (uint32_t g = threadIdx.x; g < sh_ngroups; g += blockDim.x) {
      const uint32_t i0 = gstart[g], i1 = gstart[g + 1];
      int id = 0;                                       // > 0: a row of a cotable / colocated table
      if (ids) {
        const uint8_t* e0 = recs + static_cast<size_t>(SS) * order[i0];
        const uint32_t ul0 = rec_ulen(e0, S);
        id = table_id_len(e0, ul0);
        if (id <= 0 || static_cast<uint32_t>(id) >= ul0 || e0[id] == '!') id = 0;
      }
      const bool continued = cont && g == 0;
      if (!continued && !id && row_above_cutoff(prm, recs, SS, S, order, res, i0, i1)) continue;
      st_feed += feed_row(prm, J, V.runs, V.rewrites, V.rewrite_cap, seg_lo, k, recs, SS, S, order, gstart, pvis, res, rw_slot,
                          g, id, continued, sh_ow0_state, &sh_ow0, tile);
    }
  }
  // first surviving entry of every row group: the one whose DocKey enters the file's user boundary values
  // (the group-start mark is not needed any more; its bit now carries this)
  if (prm->R.enabled) {
    for (uint32_t g = threadIdx.x; g < sh_ngroups; g += blockDim.x) {
      const uint32_t i0 = gstart[g], i1 = gstart[g + 1];
      bool done = false;
      for (uint32_t i = i0; i < i1; i++) {
        uint8_t f = res[i] & static_cast<uint8_t>(~ENT_FIRST_OF_ROW);
        if (!done && (f & ENT_KEEP)) { f |= ENT_FIRST_OF_ROW; done = true; }
        res[i] = f;
      }
    }
  }
  __syncthreads();

  // (e) descriptors in merged order
  const unsigned long long rank0 = V.tile_rank[tile] & ~TILE_CONT;
  unsigned long long st_kept = 0, st_kbytes = 0, st_vbytes = 0, st_kdel = 0, mn = ~0ull, mx = 0;
  for (uint32_t i = threadIdx.x; i < T; i += blockDim.x) {
    const uint8_t* e = recs + static_cast<size_t>(SS) * order[i];
    const uint32_t r = staged_run(e, S);
    const uint8_t f = res[i];
    Desc d;
    d.gid = V.runs[r].gid_base + staged_idx(e, S);
    d.klen = static_cast<uint16_t>(rec_ulen(e, S) + 8);
    d.flags = prm->R.enabled ? f : (f & static_cast<uint8_t>(~ENT_GROUP_START)); d.run = static_cast<uint8_t>(r);
    d.rewrite_slot = rw_slot[i];
    uint32_t vout = rec_vlen(e, S);
    if (f & ENT_VAL_TOMBSTONE) vout = 1;
    else if (f & ENT_VAL_REENCODE) { const ValueRewrite& rw = V.rewrites[rw_slot[i]]; vout = vout - rw.skip + rw.prefix_len; }
    d.vlen_out = vout;
    if ((f & ENT_KEEP) && !(f & ENT_VAL_REENCODE)) {
      // For the block encoder: bytes shared with the previous SURVIVOR's key (BlockBuilder::Add, block_builder.cc:363-365),
      // found here while both records sit in shared memory; it rides in the unused rewrite slot. 0xffff = not known (first
      // survivor of the tile, a long run of dropped entries in between, one user key a prefix of the other): k_entry_sizes
      // computes those few from the records.
      uint32_t sh = 0xffffu;
      int j = static_cast<int>(i) - 1;
      for (int steps = 0; j >= 0 && !(res[j] & ENT_KEEP) && steps < 24; steps++) j--;
      if (j >= 0 && (res[j] & ENT_KEEP)) {
        const uint8_t* p = recs + static_cast<size_t>(SS) * order[j];
        const uint32_t m = min(rec_ulen(e, S), rec_ulen(p, S));
        const uint32_t c = common_prefix_len(e, m, p, m);
        if (c < m) sh = c;
      }
      d.rewrite_slot = sh;
    }
    V.desc[rank0 + i] = d;
    if (f & ENT_KEEP) {
      st_kept++; st_kbytes += d.klen; st_vbytes += vout;
      if ((rec_suffix(e, S) & 0xff) != 1) st_kdel++;
      const unsigned long long seq = (f & ENT_ZERO_SEQ) ? 0ull : (rec_suffix(e, S) >> 8);
      mn = min(mn, seq); mx = max(mx, seq);
    }
  }
  // block-reduce stats: warp sums (one vote decides for all ten counters whether 32-bit sums are exact), per-warp
  // partials in the sort-prefix area (dead since the merge; 16 * cap >= 1 024 bytes for keys of up to 1 008 bytes), then
  // one lane per counter adds the warps and makes the tile's one global update of it. Shared-memory 64-bit atomics would
  // be compare-and-swap loops that the warps of a tile retry against each other.
  constexpr int NSTAT = 12, NWARPS = MERGE_THREADS / 32;
  unsigned long long vals[NSTAT] = {st_counted, st_hidden, st_obsolete, st_feed, st_kept, st_kbytes, st_vbytes, st_in_k, st_in_v, st_kdel, mn, mx};
  unsigned long long any_big = 0;
#pragma unroll
  for (int q = 0; q < 10; q++) any_big |= vals[q] >> 26;
  if (__any_sync(0xffffffffu, any_big != 0)) {            // giant values: 64-bit butterflies
#pragma unroll
    for (int q = 0; q < 10; q++)
      for (int o = 16; o; o >>= 1) vals[q] += __shfl_xor_sync(0xffffffffu, vals[q], o);
  } else {
#pragma unroll
    for (int q = 0; q < 10; q++) vals[q] = __reduce_add_sync(0xffffffffu, static_cast<unsigned>(vals[q]));   // one instruction each
  }
  for (int o = 16; o; o >>= 1) {
    vals[10] = min(vals[10], __shfl_xor_sync(0xffffffffu, vals[10], o));
    vals[11] = max(vals[11], __shfl_xor_sync(0xffffffffu, vals[11], o));
  }
  unsigned long long* part = pfx;                          // [NWARPS][NSTAT]
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int q = 0; q < NSTAT; q++) part[(threadIdx.x >> 5) * NSTAT + q] = vals[q];
  }
  __syncthreads();
  if (threadIdx.x < NSTAT) {
    const int q = static_cast<int>(threadIdx.x);
    unsigned long long v = part[q];
    for (int w = 1; w < NWARPS; w++) {
      const unsigned long long x = part[w * NSTAT + q];
      v = q == 10 ? min(v, x) : q == 11 ? max(v, x) : v + x;
    }
    switch (q) {
      case 0: if (v) atomicAdd(&J->n_counted, v); break;
      case 1: if (v) atomicAdd(&J->n_hidden, v); break;
      case 2: if (v) atomicAdd(&J->n_obsolete, v); break;
      case 3: if (v) atomicAdd(&J->n_feed_dropped, v); break;
      case 4: if (v) atomicAdd(&J->n_kept, v); break;
      case 5: if (v) atomicAdd(&J->out_key_bytes, v); break;
      case 6: if (v) atomicAdd(&J->out_val_bytes, v); break;
      case 7: if (v) atomicAdd(&J->in_key_bytes, v); break;
      case 8: if (v) atomicAdd(&J->in_val_bytes, v); break;
      case 9: if (v) atomicAdd(&J->n_kept_deletions, v); break;
      case 10: if (v != ~0ull) atomicMin(&J->min_seq, v); break;
      default: if (v) atomicMax(&J->max_seq, v); break;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// K4: emit. Chunked three-quantity scan (count, key bytes, value bytes) over the descriptors,
// then gather.
constexpr int EMIT_CHUNK = 2048;
constexpr int EMIT_THREADS = 256;

struct Sums3 { unsigned long long n, kb, vb; };

__global__ void __launch_bounds__(EMIT_THREADS) k_emit_sums(const Desc* desc, uint64_t N, Sums3* partial) {
  __shared__ unsigned long long sh[3];
  if (threadIdx.x < 3) sh[threadIdx.x] = 0;
  __syncthreads();
  const uint64_t base = static_cast<uint64_t>(blockIdx.x) * EMIT_CHUNK;
  unsigned long long n = 0, kb = 0, vb = 0;
  for (uint32_t j = threadIdx.x; j < EMIT_CHUNK; j += blockDim.x) {
    uint64_t i = base + j;
    if (i < N) { Desc d = desc[i]; if (d.flags & ENT_KEEP) { n++; kb += d.klen; vb += d.vlen_out; } }
  }
  for (int o = 16; o; o >>= 1) { n += __shfl_xor_sync(0xffffffffu, n, o); kb += __shfl_xor_sync(0xffffffffu, kb, o); vb += __shfl_xor_sync(0xffffffffu, vb, o); }
  if ((threadIdx.x & 31) == 0) { atomicAdd(&sh[0], n); atomicAdd(&sh[1], kb); atomicAdd(&sh[2], vb); }
  __syncthreads();
  if (threadIdx.x == 0) { partial[blockIdx.x].n = sh[0]; partial[blockIdx.x].kb = sh[1]; partial[blockIdx.x].vb = sh[2]; }
}

__global__ void __launch_bounds__(1024) k_scan_sums(Sums3* partial, uint32_t n) {
  // single CTA exclusive scan of three u64 sequences
  __shared__ unsigned long long ws[3][32];
  __shared__ unsigned long long carry[3];
  if (threadIdx.x < 3) carry[threadIdx.x] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (uint32_t base = 0; base < n; base += 1024) {
    uint32_t i = base + threadIdx.x;
    unsigned long long v[3] = {0, 0, 0};
    if (i < n) { v[0] = partial[i].n; v[1] = partial[i].kb; v[2] = partial[i].vb; }
    unsigned long long x[3] = {v[0], v[1], v[2]};
    for (int q = 0; q < 3; q++) {
      for (int o = 1; o < 32; o <<= 1) { unsigned long long y = __shfl_up_sync(0xffffffffu, x[q], o); if (lane >= o) x[q] += y; }
      if (lane == 31) ws[q][wid] = x[q];
    }
    __syncthreads();
    if (wid == 0) {
      for (int q = 0; q < 3; q++) {
        unsigned long long w = ws[q][lane];
        for (int o = 1; o < 32; o <<= 1) { unsigned long long y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
        ws[q][lane] = w;
      }
    }
    __syncthreads();
    if (i < n) {
      partial[i].n = carry[0] + (wid ? ws[0][wid - 1] : 0) + x[0] - v[0];
      partial[i].kb = carry[1] + (wid ? ws[1][wid - 1] : 0) + x[1] - v[1];
      partial[i].vb = carry[2] + (wid ? ws[2][wid - 1] : 0) + x[2] - v[2];
    }
    __syncthreads();
    if (threadIdx.x < 3) carry[threadIdx.x] += ws[threadIdx.x][31];
    __syncthreads();
  }
}

__device__ __forceinline__ void warp_copy(uint8_t* dst, const uint8_t* src, uint32_t n, int lane) {
  // dst-aligned 4-byte stores; source words assembled with a funnel shift. Reads at most 3 bytes
  // beyond src+n and 3 before src (buffers are padded by 16 bytes on both sides of the payload).
  uint32_t head = (4 - (reinterpret_cast<uintptr_t>(dst) & 3)) & 3;
  if (head > n) head = n;
  if (lane < static_cast<int>(head)) dst[lane] = src[lane];
  dst += head; src += head; n -= head;
  const uint32_t nw = n >> 2;
  const uint32_t sh = reinterpret_cast<uintptr_t>(src) & 3;
  const uint32_t* s32 = reinterpret_cast<const uint32_t*>(src - sh);
  uint32_t* d32 = reinterpret_cast<uint32_t*>(dst);
  for (uint32_t w = lane; w < nw; w += 32) {
    uint32_t lo = __ldg(s32 + w);
    if (sh) { uint32_t hi = __ldg(s32 + w + 1); lo = __funnelshift_r(lo, hi, sh * 8); }
    d32[w] = lo;
  }
  const uint32_t tail = n & 3;
  if (lane < static_cast<int>(tail)) dst[nw * 4 + lane] = src[nw * 4 + lane];
}

struct EmitView {
  const RunView* runs;
  const Desc* desc;
  const Sums3* partial;
  const ValueRewrite* rewrites;
  uint8_t* out_keys; uint64_t* out_koff;
  uint8_t* out_vals; uint64_t* out_voff;
  uint64_t N;
};

__global__ void __launch_bounds__(EMIT_THREADS) k_emit(EmitView E, int S, JobDev* J) {
  __shared__ uint32_t s_n[EMIT_CHUNK + 1];
  __shared__ uint32_t s_kb[EMIT_CHUNK + 1];
  __shared__ uint32_t s_vb[EMIT_CHUNK + 1];
  __shared__ uint32_t warp_sums[32];
  const uint64_t base = static_cast<uint64_t>(blockIdx.x) * EMIT_CHUNK;
  const Sums3 off = E.partial[blockIdx.x];
  // local exclusive scans: each thread owns EMIT_CHUNK / EMIT_THREADS consecutive descriptors
  constexpr int PER = EMIT_CHUNK / EMIT_THREADS;
  uint32_t n = 0, kb = 0, vb = 0;
  uint32_t ln[PER], lk[PER], lv[PER];
  for (int j = 0; j < PER; j++) {
    uint64_t i = base + threadIdx.x * PER + j;
    ln[j] = n; lk[j] = kb; lv[j] = vb;
    if (i < E.N) { Desc d = E.desc[i]; if (d.flags & ENT_KEEP) { n++; kb += d.klen; vb += d.vlen_out; } }
  }
  uint32_t bn = block_exclusive_scan(n, warp_sums, nullptr);
  uint32_t bk = block_exclusive_scan(kb, warp_sums, nullptr);
  uint32_t bv = block_exclusive_scan(vb, warp_sums, nullptr);
  for (int j = 0; j < PER; j++) {
    uint32_t q = threadIdx.x * PER + j;
    s_n[q] = bn + ln[j]; s_kb[q] = bk + lk[j]; s_vb[q] = bv + lv[j];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (uint32_t q = wid; q < EMIT_CHUNK; q += EMIT_THREADS / 32) {
    const uint64_t i = base + q;
    if (i >= E.N) break;
    const Desc d = E.desc[i];
    if (!(d.flags & ENT_KEEP)) continue;
    const RunView& run = E.runs[d.run];
    const uint32_t idx = d.gid - run.gid_base;
    const uint8_t* rec = run.rec + static_cast<size_t>(idx) * S;
    const uint64_t j = off.n + s_n[q];
    const uint64_t ko = off.kb + s_kb[q], vo = off.vb + s_vb[q];
    if (lane == 0) { E.out_koff[j] = ko; E.out_voff[j] = vo; }
    // key: user key bytes + 8-byte suffix
    const uint32_t ulen = d.klen - 8u;
    uint8_t* kd = E.out_keys + ko;
    for (uint32_t b = lane; b < ulen; b += 32) kd[b] = rec[b];
    if (lane < 8) {
      uint64_t suffix = rec_suffix(rec, S);
      if (d.flags & ENT_ZERO_SEQ) suffix &= 0xff;
      kd[ulen + lane] = static_cast<uint8_t>(suffix >> (8 * lane));
    }
    // value
    uint8_t* vd = E.out_vals + vo;
    const uint8_t* vs = run.data + run.val_off[idx];
    if (d.flags & ENT_VAL_TOMBSTONE) {
      if (lane == 0) vd[0] = 'X';
    } else if (d.flags & ENT_VAL_REENCODE) {
      const ValueRewrite& rw = E.rewrites[d.rewrite_slot];
      if (lane < rw.prefix_len) vd[lane] = rw.prefix[lane];
      const uint32_t rest = d.vlen_out - rw.prefix_len;
      for (uint32_t b = lane; b < rest; b += 32) vd[rw.prefix_len + b] = vs[rw.skip + b];
    } else {
      warp_copy(vd, vs, d.vlen_out, lane);
    }
  }
  (void)J;
}

// Order-sensitive digest of the emitted KV stream (test aid): per entry FNV-1a-64 over
// (klen u32, key, vlen u32, value), finalised with the entry index, summed mod 2^64.
__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33; return x;
}
__global__ void __launch_bounds__(256) k_digest(const uint8_t* keys, const uint64_t* koff, const uint8_t* vals,
                                                const uint64_t* voff, uint64_t n, JobDev* J) {
  unsigned long long acc = 0;
  for (uint64_t i = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    unsigned long long h = 1469598103934665603ull;
    const uint32_t kl = static_cast<uint32_t>(koff[i + 1] - koff[i]), vl = static_cast<uint32_t>(voff[i + 1] - voff[i]);
    for (int b = 0; b < 4; b++) { h ^= (kl >> (8 * b)) & 0xff; h *= 1099511628211ull; }
    const uint8_t* p = keys + koff[i];
    for (uint32_t b = 0; b < kl; b++) { h ^= p[b]; h *= 1099511628211ull; }
    for (int b = 0; b < 4; b++) { h ^= (vl >> (8 * b)) & 0xff; h *= 1099511628211ull; }
    p = vals + voff[i];
    for (uint32_t b = 0; b < vl; b++) { h ^= p[b]; h *= 1099511628211ull; }
    acc += mix64(h + i * 0x9e3779b97f4a7c15ull);
  }
  for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0 && acc) atomicAdd(&J->digest, acc);
}

}  // namespace ybgpu
#include "encode_kernels.cuh"
#include "ingest_kernels.cuh"
#include "snappy_kernels.cuh"   // and lz4_kernels.cuh
#include "verify_kernels.cuh"
namespace ybgpu {

// =============================================================================================
// Host orchestration
// =============================================================================================
static const char* DevErrorName(int e) {
  switch (e) {
    case DEV_ERR_BAD_BLOCK: return "bad block contents";
    case DEV_ERR_BAD_ENTRY: return "bad entry in block";
    case DEV_ERR_COMPRESSED: return "compressed block (only kNoCompression, kSnappyCompression, kLZ4Compression and kLZ4HCCompression inputs are supported)";
    case DEV_ERR_KEY_TOO_LONG: return "key longer than the engine limit";
    case DEV_ERR_IRREGULAR_RESTARTS: return "data block restart intervals are not uniform";
    case DEV_ERR_BAD_KEY: return "cannot decode DocKey/SubDocKey components";
    case DEV_ERR_UNSUPPORTED_KEY: return "key component type not supported on the GPU path";
    case DEV_ERR_TILE_OVERFLOW: return "internal error: merge tile larger than its capacity";
    case DEV_ERR_BAD_HT: return "bad DocHybridTime at the end of a key";
    case DEV_ERR_BAD_VALUE: return "cannot decode value control fields";
    case DEV_ERR_STACK_DEPTH: return "too many subkey levels";
    case DEV_ERR_UNSUPPORTED_VALUE: return "record type needs a host callback (packed row / merge / single delete)";
    case DEV_ERR_BAD_CRC: return "block checksum mismatch";
    case DEV_ERR_SHORT_KEY: return "internal key shorter than 8 bytes";
    case DEV_ERR_UNSORTED: return "input file is not sorted";
    default: return "unknown device error";
  }
}

static ybgpu_status DevErrorStatus(int e) {
  switch (e) {
    case DEV_ERR_COMPRESSED: case DEV_ERR_UNSUPPORTED_KEY: case DEV_ERR_UNSUPPORTED_VALUE:
    case DEV_ERR_TILE_OVERFLOW: case DEV_ERR_KEY_TOO_LONG: case DEV_ERR_STACK_DEPTH:
    case DEV_ERR_IRREGULAR_RESTARTS:
      return YBGPU_NOT_SUPPORTED;
    default: return YBGPU_CORRUPTION;
  }
}

// Every device allocation and free of a job goes through here: the job's own buffers, the early frees after the output
// gather and the output check's temporaries. It keeps the live blocks, the requested bytes in use (the engine's 32-byte
// pads included; the pool's rounding to its own granularity is not counted), their high-water mark and the job's
// device_memory_budget (0 = none: then nothing is checked and allocation is a plain cudaMallocAsync).
struct JobMemory {
  std::vector<std::pair<void*, size_t>> live;
  uint64_t in_use = 0, peak = 0, budget = 0;
  MemGroup* group = nullptr;           // the jobs whose bytes live at once are counted together (pipelined ranges)
  uint64_t refused = 0;                // size of the request the budget just refused (0 = none)
  static size_t Padded(size_t bytes) { return std::max<size_t>(bytes, 16) + 32; }
  bool Fits(uint64_t more) const { return !budget || (more <= budget && in_use <= budget - more); }
  cudaError_t Alloc(void** p, size_t bytes, cudaStream_t s) {
    if (!Fits(bytes)) { refused = bytes; return cudaErrorMemoryAllocation; }
    cudaError_t e = cudaMallocAsync(p, bytes, s);
    if (e != cudaSuccess) return e;
    live.emplace_back(*p, bytes);
    in_use += bytes;
    peak = std::max(peak, in_use);
    if (group) group->Change(static_cast<int64_t>(bytes));
    return cudaSuccess;
  }
  cudaError_t Free(void* p, cudaStream_t s) {
    for (size_t i = live.size(); i-- > 0;)
      if (live[i].first == p) {
        in_use -= live[i].second;
        if (group) group->Change(-static_cast<int64_t>(live[i].second));
        live.erase(live.begin() + i);
        return cudaFreeAsync(p, s);
      }
    return cudaSuccess;
  }
  void FreeAll(cudaStream_t s) {
    for (auto& a : live) cudaFreeAsync(a.first, s);
    live.clear();
    if (group) group->Change(-static_cast<int64_t>(in_use));
    in_use = 0;
  }
};

struct Engine::Impl {
  cudaStream_t stream = nullptr;
  bool owns_stream = false;            // cuda_stream == YBGPU_STREAM_PRIVATE: created in Init, destroyed with the job
  uint8_t* status_host = nullptr; uint8_t* status_dev = nullptr;   // host-mapped page for small read-backs (may be null)
  uint32_t readback_launches = 0;
  // KV-stream inputs (add_input_kv): device copies of the key bytes / offset arrays per input, entries, longest key
  struct KvInput { const uint8_t* keys; const unsigned long long* koff; const unsigned long long* voff; uint32_t n; uint32_t max_klen; std::string last_user_key; };
  std::vector<KvInput> kv;
  std::vector<std::vector<uint32_t>> cf_oids;         // per input: cotable HybridTime filters (host copies until Run)
  std::vector<std::vector<uint64_t>> cf_hts;
  uint8_t* staging_host = nullptr; uint8_t* staging_dev = nullptr;   // host-mapped staging for metadata-sized read-backs
  size_t upload_off = 0;                             // ring position of the next small upload inside the page
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  cudaEvent_t phase_ev[8] = {};
  cudaEvent_t enc_ev[2] = {};          // around the block-assembler launch (the dominant kernel of the encode phase)
  bool enc_timed = false;
  cudaEvent_t snap_ev[4] = {};         // around the output block compressor (Snappy or LZ4) and the gather of the stored blocks
  bool snap_timed = false;
  JobMemory mem;
  uint64_t image_bytes = 0, compressed_blocks = 0;   // uncompressed image the inputs added so far will need (host-known)
  JobDev* dJ = nullptr;
  JobParams* dP = nullptr;
  RunView* dRuns = nullptr;
  std::vector<RunView> runs;
  std::vector<bool> owns_data;
  std::vector<std::vector<uint64_t>> keep_off; std::vector<std::vector<uint32_t>> keep_sz;   // sources of async H2D copies
  // outputs
  uint8_t* out_keys = nullptr; uint64_t* out_koff = nullptr;
  uint8_t* out_vals = nullptr; uint64_t* out_voff = nullptr;
  uint64_t n_out = 0, out_key_bytes = 0, out_val_bytes = 0;
  JobDev hJ{};
  // K4/K5 state kept for lazy result fetches
  Desc* d_desc = nullptr; Sums3* d_partial = nullptr; ValueRewrite* d_rw = nullptr;
  bool partial_ready = false;   // d_partial holds the scanned chunk sums (computed when survivors are compacted or the KV stream is fetched)
  uint64_t N = 0; int S = 0; uint32_t n_chunks = 0;
  bool kv_emitted = false;
  Desc* d_kept = nullptr;
  uint8_t* out_file = nullptr; uint64_t out_file_len = 0;
  uint32_t n_blocks = 0; unsigned long long* d_block_off = nullptr; uint32_t* d_block_first = nullptr;
  uint8_t* d_boundary = nullptr; uint32_t boundary_stride = 0;
  EncView enc{};
  cudaStream_t copy_stream = nullptr; cudaEvent_t copy_ev = nullptr; bool copy_pending = false;
  // bloom filter blocks
  uint32_t n_filter_blocks = 0, filter_block_bytes = 0, filter_key_stride = 0;
  uint8_t* d_filters = nullptr; uint8_t* d_filter_keys = nullptr; uint32_t* d_filter_first = nullptr;
  BvOut* d_bv = nullptr;               // user boundary values (options.compute_user_boundary_values)
};

// Small device->host reads between phases (error word, counts: <= 4 KB) do not use the copy engine:
// a one-CTA kernel stores the words into a host-mapped pinned page (a posted PCIe write from the SM)
// and the host reads the page after the stream synchronises. Next to other jobs' multi-GB output
// copies a DMA read-back would queue behind them on the device->host engine.
// KV-stream inputs (ybgpu_job_add_input_kv: the contents of a memtable for a flush, rocksdb/db/builder.cc:119-318, or any
// sorted run a caller holds in memory): internal keys back to back with an offset array, values likewise. One thread per
// entry writes the fixed-stride key record the rest of the pipeline works on; the values stay where they are.
__global__ void __launch_bounds__(256) k_records_from_kv(const uint8_t* keys, const unsigned long long* koff, const unsigned long long* voff,
                                                         const uint8_t* vals, uint32_t n, int S, uint8_t* rec, uint64_t* val_off, JobDev* J) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned long long k0 = koff[i], k1 = koff[i + 1], v0 = voff[i], v1 = voff[i + 1];
    uint8_t* r = rec + static_cast<size_t>(i) * S;
    if (k1 < k0 + 8 || k1 - k0 - 8 > static_cast<unsigned long long>(S - 16) || v1 < v0 || v1 - v0 >= (1ull << 32)) {
      dev_fail(J, k1 < k0 + 8 ? DEV_ERR_SHORT_KEY : DEV_ERR_BAD_ENTRY, i);
      for (int b = 0; b < S; b++) r[b] = 0;
      val_off[i] = 0;
      continue;
    }
    const uint32_t ulen = static_cast<uint32_t>(k1 - k0 - 8), vlen = static_cast<uint32_t>(v1 - v0);
    const uint8_t* kp = keys + k0;
    for (int b = 0; b < S - 16; b++) r[b] = static_cast<uint32_t>(b) < ulen ? kp[b] : 0;
    uint64_t suffix = 0;
    for (int b = 7; b >= 0; b--) suffix = (suffix << 8) | kp[ulen + b];
    uint4 tr;
    tr.x = static_cast<uint32_t>(suffix); tr.y = static_cast<uint32_t>(suffix >> 32);
    tr.z = ulen | (static_cast<uint32_t>(vlen ? vals[v0] : 0) << 16);
    tr.w = vlen;
    *reinterpret_cast<uint4*>(r + S - 16) = tr;
    val_off[i] = v0;
  }
}

__global__ void k_readback(uint8_t* dst_mapped, const uint8_t* src, uint32_t n) {
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) dst_mapped[i] = src[i];
  __threadfence_system();
}
constexpr size_t STATUS_READ_BYTES = 4096;             // [0, 4096): read-backs; the rest: a ring of small parameter uploads
constexpr size_t STATUS_PAGE_BYTES = 65536;
struct StatusPage { uint8_t* host = nullptr; uint8_t* dev = nullptr; };
static std::mutex g_status_mu;
static std::vector<StatusPage> g_status_free;          // process-wide: cudaHostAlloc is expensive
static cudaError_t AcquireStatusPage(StatusPage* p) {
  {
    std::lock_guard<std::mutex> lock(g_status_mu);
    if (!g_status_free.empty()) { *p = g_status_free.back(); g_status_free.pop_back(); return cudaSuccess; }
  }
  void* h = nullptr; void* d = nullptr;
  cudaError_t e = cudaHostAlloc(&h, STATUS_PAGE_BYTES, cudaHostAllocMapped | cudaHostAllocPortable);
  if (e != cudaSuccess) return e;
  e = cudaHostGetDevicePointer(&d, h, 0);
  if (e != cudaSuccess) { cudaFreeHost(h); return e; }
  p->host = static_cast<uint8_t*>(h); p->dev = static_cast<uint8_t*>(d);
  return cudaSuccess;
}
static void ReleaseStatusPage(const StatusPage& p) {
  if (!p.host) return;
  std::lock_guard<std::mutex> lock(g_status_mu);
  g_status_free.push_back(p);
}
// Metadata-sized device -> host reads (block offsets, boundary keys, bloom filter blocks: megabytes per job) bypass the
// copy engine as well: in a pipelined compaction the D2H engine is busy with the neighbours' output files for tens of
// milliseconds at a stretch, and a job cannot size / place its own output before it has these arrays. A kernel stores
// them into host-mapped pinned staging memory (posted PCIe writes from the SMs), the host copies them out of there.
constexpr size_t STAGING_BYTES = 8u << 20;
struct Staging { uint8_t* host = nullptr; uint8_t* dev = nullptr; };
static std::vector<Staging> g_staging_free;            // process-wide, guarded by g_status_mu
static cudaError_t AcquireStaging(Staging* p) {
  {
    std::lock_guard<std::mutex> lock(g_status_mu);
    if (!g_staging_free.empty()) { *p = g_staging_free.back(); g_staging_free.pop_back(); return cudaSuccess; }
  }
  void* h = nullptr; void* d = nullptr;
  cudaError_t e = cudaHostAlloc(&h, STAGING_BYTES, cudaHostAllocMapped | cudaHostAllocPortable);
  if (e != cudaSuccess) return e;
  e = cudaHostGetDevicePointer(&d, h, 0);
  if (e != cudaSuccess) { cudaFreeHost(h); return e; }
  p->host = static_cast<uint8_t*>(h); p->dev = static_cast<uint8_t*>(d);
  return cudaSuccess;
}
static void ReleaseStaging(const Staging& p) {
  if (!p.host) return;
  std::lock_guard<std::mutex> lock(g_status_mu);
  g_staging_free.push_back(p);
}
// rows of `row_bytes` bytes, `src_pitch` apart in device memory, packed back to back in the destination
__global__ void __launch_bounds__(256) k_copy_out(uint8_t* dst_mapped, const uint8_t* src, size_t row_bytes, size_t src_pitch, size_t rows) {
  const size_t total = row_bytes * rows;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  if (src_pitch == row_bytes && ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst_mapped)) & 15) == 0) {
    const size_t nv = total >> 4;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < nv; i += stride)
      reinterpret_cast<uint4*>(dst_mapped)[i] = reinterpret_cast<const uint4*>(src)[i];
    for (size_t i = (nv << 4) + blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total; i += stride) dst_mapped[i] = src[i];
  } else {
    // pitched rows (bloom filter blocks): a CTA walks whole rows, no division per byte
    for (size_t r = blockIdx.x; r < rows; r += gridDim.x)
      for (size_t c = threadIdx.x; c < row_bytes; c += blockDim.x) dst_mapped[r * row_bytes + c] = src[r * src_pitch + c];
  }
  __threadfence_system();
}

static bool ZeroCopyStatusEnabled() {
  const char* e = getenv("YBGPU_ZC_STATUS");
  return e ? atoi(e) != 0 : true;
}

Engine::Engine(const ybgpu_job_options& o) : opt_(o), impl_(new Impl) {
  if (o.largest_user_key && o.has_largest_user_key) largest_.assign(o.largest_user_key, o.largest_user_key + o.largest_user_key_len);
  if (o.key_bounds_lower_len) lower_.assign(o.key_bounds_lower, o.key_bounds_lower + o.key_bounds_lower_len);
  if (o.key_bounds_upper_len) upper_.assign(o.key_bounds_upper, o.key_bounds_upper + o.key_bounds_upper_len);
  if (o.range_lower_len) range_lower_.assign(o.range_lower, o.range_lower + o.range_lower_len);
  if (o.range_upper_len) range_upper_.assign(o.range_upper, o.range_upper + o.range_upper_len);
  opt_.range_lower = nullptr; opt_.range_upper = nullptr;
  opt_.largest_user_key = nullptr; opt_.key_bounds_lower = nullptr; opt_.key_bounds_upper = nullptr;
  memset(&stats_, 0, sizeof(stats_));
  impl_->mem.budget = o.device_memory_budget;
}

Engine::~Engine() {
  if (impl_) {
    cudaSetDevice(opt_.device);
    if (impl_->copy_pending) cudaStreamSynchronize(impl_->copy_stream);   // before the output buffer returns to the pool
    // a job abandoned before Run() may still have input DMAs queued that read the caller's buffers
    if (!ran_ && !impl_->runs.empty()) cudaStreamSynchronize(impl_->stream);
    impl_->mem.FreeAll(impl_->stream);
    if (impl_->ev0) cudaEventDestroy(impl_->ev0);
    if (impl_->ev1) cudaEventDestroy(impl_->ev1);
    if (impl_->copy_stream) cudaStreamDestroy(impl_->copy_stream);
    if (impl_->copy_ev) cudaEventDestroy(impl_->copy_ev);
    for (auto& e : impl_->enc_ev) if (e) cudaEventDestroy(e);
    for (auto& e : impl_->snap_ev) if (e) cudaEventDestroy(e);
    for (auto& e : impl_->phase_ev) if (e) cudaEventDestroy(e);
    if (impl_->staging_host) { Staging st; st.host = impl_->staging_host; st.dev = impl_->staging_dev; ReleaseStaging(st); }   // every read through it was synchronous
    if (impl_->status_host) {
      cudaStreamSynchronize(impl_->stream);              // no read-back kernel may still target the page
      StatusPage pg; pg.host = impl_->status_host; pg.dev = impl_->status_dev;
      ReleaseStatusPage(pg);
    }
    if (impl_->owns_stream && impl_->stream) cudaStreamDestroy(impl_->stream);   // the queued frees complete first
    delete impl_;
  }
}

ybgpu_status Engine::Fail(ybgpu_status s, const std::string& msg) { error_ = msg; return s; }

static std::string BudgetMessage(uint64_t need, uint64_t in_use, uint64_t budget) {
  return std::string(kBudgetExceeded) + ": need " + std::to_string(need) + ", in use " + std::to_string(in_use) + ", budget " +
         std::to_string(budget);
}

ybgpu_status Engine::FailCuda(const char* expr, int e) {
  JobMemory& M = impl_->mem;
  if (M.refused) {
    const uint64_t need = M.refused;
    M.refused = 0;
    cudaStreamSynchronize(impl_->stream);                 // nothing the failed job queued is still running when it returns
    return Fail(YBGPU_RUNTIME_ERROR, BudgetMessage(need, M.in_use, M.budget));
  }
  return Fail(YBGPU_RUNTIME_ERROR, std::string(expr) + ": " + cudaGetErrorString(static_cast<cudaError_t>(e)));
}

// Host-known bytes (`more` beyond what the job holds) checked against the budget before anything is uploaded.
ybgpu_status Engine::CheckBudgetBeforeUpload(uint64_t more) {
  const JobMemory& M = impl_->mem;
  if (M.Fits(more)) return YBGPU_OK;
  return Fail(YBGPU_NOT_SUPPORTED, BudgetMessage(more, M.in_use, M.budget) + " (inputs and their uncompressed image, before upload)");
}

void Engine::JoinMemGroup(MemGroup* group) {
  impl_->mem.group = group;
  group->Change(static_cast<int64_t>(impl_->mem.in_use));
}

ybgpu_job_stats& Engine::stats() {
  stats_.device_bytes_peak = impl_->mem.peak;
  return stats_;
}

// Stream-ordered allocation from the device's default memory pool (release threshold raised to
// "never" in Init), so steady-state jobs reuse HBM instead of paying cudaMalloc/cudaFree.
static thread_local cudaStream_t g_alloc_stream = nullptr;
template <typename T>
static cudaError_t DevAlloc(JobMemory* mem, T** out, size_t count) {
  void* p = nullptr;
  cudaError_t e = mem->Alloc(&p, JobMemory::Padded(count * sizeof(T)), g_alloc_stream);
  if (e == cudaSuccess) *out = reinterpret_cast<T*>(p);
  return e;
}


// Bulk host<->device copies are issued in chunks: a copy engine serves its queues copy by copy, so a
// multi-GB cudaMemcpyAsync of one job would hold every small copy of the jobs running beside it
// (status words, block counts, parameters: ~10 round trips per job) for tens of milliseconds.
static size_t CopyChunkBytes() {
  const char* e = getenv("YBGPU_COPY_CHUNK_MB");          // read per bulk copy (a handful per job)
  const long mb = e ? atol(e) : 32;
  return mb > 0 ? static_cast<size_t>(mb) << 20 : ~static_cast<size_t>(0);
}
static cudaError_t ChunkedCopyAsync(void* dst, const void* src, size_t len, cudaMemcpyKind kind, cudaStream_t stream) {
  const size_t chunk = CopyChunkBytes();
  for (size_t off = 0; off < len; off += chunk) {
    cudaError_t e = cudaMemcpyAsync(static_cast<uint8_t*>(dst) + off, static_cast<const uint8_t*>(src) + off, std::min(chunk, len - off), kind, stream);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

ybgpu_status Engine::Init() {
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return Fail(YBGPU_RUNTIME_ERROR, std::string("no usable CUDA device: ") + cudaGetErrorString(e) +
                                         " (this engine has no CPU fallback)");
  if (opt_.device < 0 || opt_.device >= ndev) return Fail(YBGPU_INVALID_ARGUMENT, "bad device ordinal");
  CUDA_TRY(cudaSetDevice(opt_.device));
  if (opt_.cuda_stream == YBGPU_STREAM_PRIVATE) {
    // jobs that run concurrently on one device (subcompactions, several tablets) must not meet on the
    // legacy default stream: each gets its own non-blocking stream
    CUDA_TRY(cudaStreamCreateWithFlags(&impl_->stream, cudaStreamNonBlocking));
    impl_->owns_stream = true;
  } else {
    impl_->stream = reinterpret_cast<cudaStream_t>(opt_.cuda_stream);   // NULL = legacy default stream
  }
  g_alloc_stream = impl_->stream;
  {
    cudaMemPool_t pool;
    CUDA_TRY(cudaDeviceGetDefaultMemPool(&pool, opt_.device));
    uint64_t thr = ~0ull;
    CUDA_TRY(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
    // Never satisfy an allocation with memory whose free is still pending on ANOTHER stream: the pool would make this
    // job's stream wait for that stream's queued work — in a pipelined compaction that is a neighbour's multi-GB output
    // copy, and this job's kernels would sit behind it. Memory whose free
    // has completed is still reused; otherwise the pool grows.
    int off = 0;
    CUDA_TRY(cudaMemPoolSetAttribute(pool, cudaMemPoolReuseAllowInternalDependencies, &off));
  }
  if (ZeroCopyStatusEnabled()) {
    StatusPage pg;
    CUDA_TRY(AcquireStatusPage(&pg));
    impl_->status_host = pg.host; impl_->status_dev = pg.dev;
  }
  CUDA_TRY(cudaEventCreate(&impl_->ev0));
  CUDA_TRY(cudaEventCreate(&impl_->ev1));
  for (auto& e : impl_->phase_ev) CUDA_TRY(cudaEventCreate(&e));
  for (auto& e : impl_->enc_ev) CUDA_TRY(cudaEventCreate(&e));
  CUDA_TRY(DevAlloc(&impl_->mem, &impl_->dJ, 1));
  CUDA_TRY(DevAlloc(&impl_->mem, &impl_->dP, 1));
  CUDA_TRY(DevAlloc(&impl_->mem, &impl_->dRuns, MAX_RUNS));
  return YBGPU_OK;
}

ybgpu_status Engine::AddInput(const uint8_t* data, uint64_t len, const ybgpu_block_handle* handles, uint64_t nh,
                              int key_encoding, uint64_t ht_filter, bool on_device) {
  if (ran_) return Fail(YBGPU_ILLEGAL_STATE, "add_input after run");
  if (impl_->runs.size() >= MAX_RUNS) return Fail(YBGPU_NOT_SUPPORTED, "too many input files");
  if (!impl_->kv.empty()) return Fail(YBGPU_NOT_SUPPORTED, "KV-stream inputs and table-file inputs cannot be mixed in one job");
  if (key_encoding != YBGPU_KEY_ENCODING_SHARED_PREFIX && key_encoding != YBGPU_KEY_ENCODING_THREE_SHARED_PARTS)
    return Fail(YBGPU_INVALID_ARGUMENT, "unknown data block key encoding");
  if (nh >= (1ull << 32)) return Fail(YBGPU_NOT_SUPPORTED, "too many data blocks in one file");
  CUDA_TRY(cudaSetDevice(opt_.device));
  g_alloc_stream = impl_->stream;
  for (uint64_t i = 0; i < nh; i++) {
    // offset + size + 5 <= len without wrapping on corrupt (huge) handles
    if (handles[i].offset > len || handles[i].size > len - handles[i].offset || len - handles[i].offset - handles[i].size < 5)
      return Fail(YBGPU_CORRUPTION, "block handle outside the data file");
    if (handles[i].size >= (1ull << 31)) return Fail(YBGPU_NOT_SUPPORTED, "data block too large");
  }
  if (impl_->mem.budget) {
    // this input's device copy and handle arrays, and — once any input block is stored compressed — the uncompressed image
    // of every input (a file already in device memory is not read on the host: its image is not known before run)
    uint64_t comp = 0;
    const uint64_t img = on_device ? 0 : host::UncompressedImageBytes(data, handles, nh, &comp);
    uint64_t more = (on_device ? 0 : JobMemory::Padded(len + 64)) + JobMemory::Padded(nh * 8) + JobMemory::Padded(nh * 4) +
                    JobMemory::Padded((nh + 1) * 4);
    if (impl_->compressed_blocks + comp) more += JobMemory::Padded(impl_->image_bytes + img + 96);
    if (ybgpu_status s = CheckBudgetBeforeUpload(more)) return s;
    impl_->image_bytes += img; impl_->compressed_blocks += comp;
  }
  RunView rv{};
  if (on_device) {
    rv.data = data;
  } else {
    uint8_t* d = nullptr;
    CUDA_TRY(DevAlloc(&impl_->mem, &d, len + 64));
    // 16 bytes of zero padding on both sides so word-granular copies may over-read
    CUDA_TRY(cudaMemsetAsync(d, 0, 16, impl_->stream));
    CUDA_TRY(ChunkedCopyAsync(d + 16, data, len, cudaMemcpyHostToDevice, impl_->stream));
    CUDA_TRY(cudaMemsetAsync(d + 16 + len, 0, 16, impl_->stream));
    rv.data = d + 16;
    stats_.h2d_bytes += len;
  }
  // handle arrays stay alive in the job so that no stream synchronisation is needed here: the H2D
  // copies of all input files queue back to back and Run() simply follows them on the stream
  impl_->keep_off.emplace_back(nh); impl_->keep_sz.emplace_back(nh);
  std::vector<uint64_t>& off = impl_->keep_off.back(); std::vector<uint32_t>& sz = impl_->keep_sz.back();
  for (uint64_t i = 0; i < nh; i++) { off[i] = handles[i].offset; sz[i] = static_cast<uint32_t>(handles[i].size); }
  uint64_t* doff = nullptr; uint32_t* dsz = nullptr; uint32_t* dcnt = nullptr;
  CUDA_TRY(DevAlloc(&impl_->mem, &doff, nh)); CUDA_TRY(DevAlloc(&impl_->mem, &dsz, nh));
  CUDA_TRY(DevAlloc(&impl_->mem, &dcnt, nh + 1));
  CUDA_TRY(cudaMemcpyAsync(doff, off.data(), nh * 8, cudaMemcpyHostToDevice, impl_->stream));
  CUDA_TRY(cudaMemcpyAsync(dsz, sz.data(), nh * 4, cudaMemcpyHostToDevice, impl_->stream));
  rv.blk_off = doff; rv.blk_size = dsz; rv.blk_count = dcnt; rv.nb = static_cast<uint32_t>(nh);
  rv.ht_filter = ht_filter;
  rv.key_encoding = static_cast<uint32_t>(key_encoding);
  impl_->runs.push_back(rv);
  impl_->cf_oids.emplace_back(); impl_->cf_hts.emplace_back();
  return YBGPU_OK;
}

ybgpu_status Engine::SetCotableFilters(const uint32_t* db_oids, const uint64_t* hybrid_times, uint32_t n) {
  if (ran_) return Fail(YBGPU_ILLEGAL_STATE, "set_cotable_filters after run");
  if (impl_->runs.empty()) return Fail(YBGPU_ILLEGAL_STATE, "set_cotable_filters before any input");
  if (n && (!db_oids || !hybrid_times)) return Fail(YBGPU_INVALID_ARGUMENT, "null cotable filter arrays");
  for (uint32_t i = 1; i < n; i++)
    if (db_oids[i - 1] >= db_oids[i]) return Fail(YBGPU_INVALID_ARGUMENT, "cotable filter database oids must be strictly increasing");
  impl_->cf_oids.back().assign(db_oids, db_oids + n);
  impl_->cf_hts.back().assign(hybrid_times, hybrid_times + n);
  return YBGPU_OK;
}

ybgpu_status Engine::AddInputKv(const uint8_t* keys, const uint64_t* key_offsets, const uint8_t* values, const uint64_t* value_offsets, uint64_t n) {
  Impl& I = *impl_;
  if (ran_) return Fail(YBGPU_ILLEGAL_STATE, "add_input after run");
  if (I.runs.size() >= MAX_RUNS) return Fail(YBGPU_NOT_SUPPORTED, "too many input files");
  if (I.kv.size() != I.runs.size()) return Fail(YBGPU_NOT_SUPPORTED, "KV-stream inputs and table-file inputs cannot be mixed in one job");
  if (n >= (1ull << 32)) return Fail(YBGPU_NOT_SUPPORTED, "more than 2^32 entries in one input");
  if (n && (!keys || !key_offsets || !value_offsets)) return Fail(YBGPU_INVALID_ARGUMENT, "null argument");
  CUDA_TRY(cudaSetDevice(opt_.device));
  g_alloc_stream = I.stream;
  const uint64_t kbytes = n ? key_offsets[n] : 0, vbytes = n ? value_offsets[n] : 0;
  uint32_t max_klen = 0;
  for (uint64_t i = 0; i < n; i++) {
    if (key_offsets[i + 1] < key_offsets[i] + 8 || value_offsets[i + 1] < value_offsets[i]) return Fail(YBGPU_INVALID_ARGUMENT, "bad key / value offsets");
    max_klen = std::max<uint32_t>(max_klen, static_cast<uint32_t>(std::min<uint64_t>(key_offsets[i + 1] - key_offsets[i], 0xffffffffu)));
  }
  if (I.mem.budget) {
    const uint64_t more = JobMemory::Padded(kbytes + 16) + JobMemory::Padded(vbytes + 64) + 2 * JobMemory::Padded((n + 1) * 8) +
                          JobMemory::Padded(4);
    if (ybgpu_status s = CheckBudgetBeforeUpload(more)) return s;
  }
  uint8_t* dk = nullptr; uint8_t* dv = nullptr; unsigned long long* dko = nullptr; unsigned long long* dvo = nullptr; uint32_t* dcnt = nullptr;
  CUDA_TRY(DevAlloc(&I.mem, &dk, kbytes + 16));
  CUDA_TRY(DevAlloc(&I.mem, &dv, vbytes + 64));
  CUDA_TRY(DevAlloc(&I.mem, &dko, n + 1)); CUDA_TRY(DevAlloc(&I.mem, &dvo, n + 1)); CUDA_TRY(DevAlloc(&I.mem, &dcnt, 1));
  CUDA_TRY(cudaMemsetAsync(dv, 0, 16, I.stream));
  if (kbytes) CUDA_TRY(ChunkedCopyAsync(dk, keys, kbytes, cudaMemcpyHostToDevice, I.stream));
  if (vbytes) CUDA_TRY(ChunkedCopyAsync(dv + 16, values, vbytes, cudaMemcpyHostToDevice, I.stream));
  CUDA_TRY(cudaMemsetAsync(dv + 16 + vbytes, 0, 16, I.stream));
  static const uint64_t zero_off[1] = {0};
  CUDA_TRY(ChunkedCopyAsync(dko, n ? key_offsets : zero_off, (n + 1) * 8, cudaMemcpyHostToDevice, I.stream));
  CUDA_TRY(ChunkedCopyAsync(dvo, n ? value_offsets : zero_off, (n + 1) * 8, cudaMemcpyHostToDevice, I.stream));
  stats_.h2d_bytes += kbytes + vbytes + 16 * (n + 1);
  RunView rv{};
  rv.data = dv + 16; rv.blk_off = nullptr; rv.blk_size = nullptr; rv.blk_count = dcnt; rv.nb = 0;
  rv.ht_filter = HT_FILTER_NONE; rv.key_encoding = YBGPU_KEY_ENCODING_SHARED_PREFIX;
  I.runs.push_back(rv);
  I.cf_oids.emplace_back(); I.cf_hts.emplace_back();
  Impl::KvInput ki{dk, dko, dvo, static_cast<uint32_t>(n), max_klen, std::string()};
  if (n) ki.last_user_key.assign(reinterpret_cast<const char*>(keys + key_offsets[n - 1]), key_offsets[n] - key_offsets[n - 1] - 8);
  I.kv.push_back(ki);
  return YBGPU_OK;
}

ybgpu_status Engine::WaitInputs() {
  CUDA_TRY(cudaSetDevice(opt_.device));
  CUDA_TRY(cudaStreamSynchronize(impl_->stream));
  return YBGPU_OK;
}

static int GridFor(uint64_t work_items, int threads, int sms) {
  uint64_t blocks = (work_items + threads - 1) / threads;
  uint64_t cap = static_cast<uint64_t>(sms) * 16;
  return static_cast<int>(std::max<uint64_t>(1, std::min(blocks, cap)));
}

// Device -> host read of a few words followed by a stream synchronisation (see k_readback).
ybgpu_status Engine::ReadSmall(void* host_dst, const void* dev_src, size_t n) {
  Impl& I = *impl_;
  if (I.status_host && n <= STATUS_READ_BYTES) {
    k_readback<<<1, 128, 0, I.stream>>>(I.status_dev, static_cast<const uint8_t*>(dev_src), static_cast<uint32_t>(n));
    I.readback_launches++;
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(I.stream));
    memcpy(host_dst, I.status_host, n);
    return YBGPU_OK;
  }
  CUDA_TRY(cudaMemcpyAsync(host_dst, dev_src, n, cudaMemcpyDeviceToHost, I.stream));
  CUDA_TRY(cudaStreamSynchronize(I.stream));
  return YBGPU_OK;
}

// Small host -> device parameter blocks (run table, job parameters, prefix tables: ~a dozen per job, < 8 KB each) go
// through the host-mapped page as well: a host -> device DMA would queue on the copy engine behind the bulk input
// copies of the jobs running beside this one (tens of milliseconds each in a pipelined compaction), and every one of
// them sits on the job's critical path. The bytes are staged in a ring inside the page and copied by one small CTA.
ybgpu_status Engine::UploadSmall(void* dev_dst, const void* host_src, size_t n) {
  Impl& I = *impl_;
  const size_t need = (n + 15) & ~static_cast<size_t>(15);
  if (!I.status_host || need > STATUS_PAGE_BYTES - STATUS_READ_BYTES) {
    CUDA_TRY(cudaMemcpyAsync(dev_dst, host_src, n, cudaMemcpyHostToDevice, I.stream));
    return YBGPU_OK;
  }
  if (I.upload_off < STATUS_READ_BYTES) I.upload_off = STATUS_READ_BYTES;
  size_t ring_end = STATUS_PAGE_BYTES;
  if (const char* e = getenv("YBGPU_UPLOAD_RING_BYTES")) {         // tests: a small ring wraps after a few uploads
    const long v = atol(e);
    if (v > 0) ring_end = std::min<size_t>(STATUS_PAGE_BYTES, STATUS_READ_BYTES + std::max<size_t>(static_cast<size_t>(v), need));
  }
  if (I.upload_off + need > ring_end) {
    CUDA_TRY(cudaStreamSynchronize(I.stream));           // every earlier upload has been consumed
    I.upload_off = STATUS_READ_BYTES;
  }
  memcpy(I.status_host + I.upload_off, host_src, n);
  k_readback<<<1, 128, 0, I.stream>>>(static_cast<uint8_t*>(dev_dst), I.status_dev + I.upload_off, static_cast<uint32_t>(n));
  I.readback_launches++;
  CUDA_TRY(cudaGetLastError());
  I.upload_off += need;
  return YBGPU_OK;
}

ybgpu_status Engine::ReadViaMapped(void* host_dst, const void* dev_src, size_t row_bytes, size_t src_pitch, size_t rows) {
  Impl& I = *impl_;
  if (!row_bytes || !rows) return YBGPU_OK;
  if (!I.status_host || row_bytes > STAGING_BYTES) {      // zero-copy reads disabled (A/B switch): the copy engine
    if (src_pitch == row_bytes) CUDA_TRY(cudaMemcpyAsync(host_dst, dev_src, row_bytes * rows, cudaMemcpyDeviceToHost, I.stream));
    else CUDA_TRY(cudaMemcpy2DAsync(host_dst, row_bytes, dev_src, src_pitch, row_bytes, rows, cudaMemcpyDeviceToHost, I.stream));
    CUDA_TRY(cudaStreamSynchronize(I.stream));
    return YBGPU_OK;
  }
  if (!I.staging_host) {
    Staging st;
    CUDA_TRY(AcquireStaging(&st));
    I.staging_host = st.host; I.staging_dev = st.dev;
  }
  const size_t rows_per = std::max<size_t>(1, STAGING_BYTES / row_bytes);
  for (size_t r0 = 0; r0 < rows; r0 += rows_per) {
    const size_t nr = std::min(rows_per, rows - r0);
    const size_t bytes = nr * row_bytes;
    const int grid = src_pitch == row_bytes ? static_cast<int>(std::min<size_t>(64, (bytes + 65535) / 65536)) : static_cast<int>(std::min<size_t>(64, nr));
    k_copy_out<<<std::max(grid, 1), 256, 0, I.stream>>>(I.staging_dev, static_cast<const uint8_t*>(dev_src) + r0 * src_pitch, row_bytes, src_pitch, nr);
    I.readback_launches++;
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(I.stream));
    memcpy(static_cast<uint8_t*>(host_dst) + r0 * row_bytes, I.staging_host, bytes);
  }
  return YBGPU_OK;
}

ybgpu_status Engine::CheckDeviceError(const char* phase) {
  Impl& I = *impl_;
  if (ybgpu_status s = ReadSmall(&I.hJ, I.dJ, sizeof(JobDev))) return s;
  if (I.hJ.error) {
    char buf[256];
    snprintf(buf, sizeof(buf), "%s (%s, at block/tile %u)", DevErrorName(I.hJ.error), phase, I.hJ.error_where);
    return Fail(DevErrorStatus(I.hJ.error), buf);
  }
  return YBGPU_OK;
}

// Per-device one-time state (SM count, CRC tables in device memory), shared by every job of the
// process; jobs may run concurrently on different host threads, so it is built under a lock and
// the table kernels are complete before any job proceeds.
static cudaError_t EnsureDeviceTables(int device, cudaStream_t stream, int* sms) {
  static std::mutex dev_init_mu;
  static int sm_count[64] = {};
  static bool crc_ready[64] = {};
  std::lock_guard<std::mutex> lock(dev_init_mu);
  cudaError_t e;
  // cudaGetDeviceProperties costs milliseconds per call; one attribute, cached per device.
  if (!sm_count[device & 63] && (e = cudaDeviceGetAttribute(&sm_count[device & 63], cudaDevAttrMultiProcessorCount, device)) != cudaSuccess) return e;
  if (!crc_ready[device & 63]) {
    k_crc_init<<<1, 256, 0, stream>>>();
    k_crc_init_xpow<<<(CRC_XPOW_TABLE + 256) / 256, 256, 0, stream>>>();
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
    crc_ready[device & 63] = true;
  }
  *sms = sm_count[device & 63];
  return cudaSuccess;
}

ybgpu_status Engine::Run(const volatile int32_t* shutting_down) {
  if (ran_) return Fail(YBGPU_ILLEGAL_STATE, "job already ran");
  Impl& I = *impl_;
  if (I.compressed_blocks)                                // counted only under a budget: the uncompressed image comes first
    if (ybgpu_status s = CheckBudgetBeforeUpload(JobMemory::Padded(I.image_bytes + 96))) return s;
  const bool trace = getenv("YBGPU_TRACE") != nullptr;
  auto t_prev = std::chrono::steady_clock::now();
  CUDA_TRY(cudaSetDevice(opt_.device));
  g_alloc_stream = I.stream;
  int sms = 0;
  CUDA_TRY(EnsureDeviceTables(opt_.device, I.stream, &sms));
  const int k = static_cast<int>(I.runs.size());
  // the yield point sits where the shutdown flag is polled: between kernel phases
  auto shutdown = [&]() {
    if (opt_.yield_fn) opt_.yield_fn(opt_.yield_ctx);
    return shutting_down && *shutting_down;
  };
  uint32_t launches = 0;

  CUDA_TRY(cudaMemsetAsync(I.dJ, 0, sizeof(JobDev), I.stream));
  {
    JobDev init{}; init.min_seq = ~0ull;
    if (ybgpu_status us = UploadSmall(I.dJ, &init, sizeof(init))) return us;
  }
  CUDA_TRY(cudaEventRecord(I.ev0, I.stream));
  uint32_t phase_launch_mark[8] = {};
  int phase = 0;
  auto tick = [&](const char* what) {
    if (!trace) return;
    cudaStreamSynchronize(I.stream);
    auto now = std::chrono::steady_clock::now();
    fprintf(stderr, "[ybgpu trace] %-14s %8.3f ms (host wall, after stream sync)\n", what, std::chrono::duration<double, std::milli>(now - t_prev).count());
    t_prev = now;
  };
  tick("setup");
  auto end_phase = [&]() -> cudaError_t {
    phase_launch_mark[phase] = launches;
    return cudaEventRecord(I.phase_ev[phase++], I.stream);
  };

  // ---- K0/K1: one fused pass (k_ingest: TMA-staged blocks, checksum verification, value CRCs, entry counts,
  // key records) when every input is shared-prefix encoded; otherwise, or when the fused kernel meets something
  // it does not take, the general kernels: k_crc_blocks (verify), k_prepass, k_decode_all, k_value_crc.
  uint32_t* d_totals = nullptr;
  CUDA_TRY(DevAlloc(&I.mem, &d_totals, static_cast<size_t>(k) + 1));
  std::vector<uint32_t> blk_base(k + 1, 0);
  for (int r = 0; r < k; r++) blk_base[r + 1] = blk_base[r] + I.runs[r].nb;
  uint32_t* d_blk_base = nullptr;
  CUDA_TRY(DevAlloc(&I.mem, &d_blk_base, static_cast<size_t>(k) + 1));
  for (int r = 0; r < k; r++) {
    const size_t n = I.cf_oids[r].size();
    if (!n || I.runs[r].cf_n) continue;
    uint32_t* d_oid = nullptr; uint64_t* d_ht = nullptr;
    CUDA_TRY(DevAlloc(&I.mem, &d_oid, n)); CUDA_TRY(DevAlloc(&I.mem, &d_ht, n));
    if (ybgpu_status us = UploadSmall(d_oid, I.cf_oids[r].data(), 4 * n)) return us;
    if (ybgpu_status us = UploadSmall(d_ht, I.cf_hts[r].data(), 8 * n)) return us;
    I.runs[r].cf_oid = d_oid; I.runs[r].cf_ht = d_ht; I.runs[r].cf_n = static_cast<uint32_t>(n);
  }
  if (ybgpu_status us = UploadSmall(d_blk_base, blk_base.data(), 4 * (static_cast<size_t>(k) + 1))) return us;
  if (ybgpu_status us = UploadSmall(I.dRuns, I.runs.data(), sizeof(RunView) * k)) return us;
  RangeDev* d_range = nullptr;
  if (!range_lower_.empty() || !range_upper_.empty()) {
    if (range_lower_.size() > 255 || range_upper_.size() > 255) return Fail(YBGPU_NOT_SUPPORTED, "range bounds longer than 255 bytes");
    RangeDev hr{};
    hr.lower_len = static_cast<uint32_t>(range_lower_.size()); memcpy(hr.lower, range_lower_.data(), range_lower_.size());
    hr.upper_len = static_cast<uint32_t>(range_upper_.size()); memcpy(hr.upper, range_upper_.data(), range_upper_.size());
    CUDA_TRY(DevAlloc(&I.mem, &d_range, 1));
    if (ybgpu_status us = UploadSmall(d_range, &hr, sizeof(hr))) return us;
  }
  uint64_t N = 0;
  uint32_t max_ikey = 0;
  int Sfinal = 32;
  bool ingested = false;
  bool try_ingest = blk_base[k] > 0 && getenv("YBGPU_NO_INGEST") == nullptr;
  for (int r = 0; r < k; r++) try_ingest = try_ingest && I.runs[r].key_encoding == 1;
  if (!I.kv.empty()) {
    // ---- KV-stream inputs: no blocks to verify or decode; records straight from the key arrays, value CRCs for the
    // block encoder from the value arrays
    try_ingest = false;
    for (int r = 0; r < k; r++) {
      I.runs[r].n_entries = I.kv[r].n;
      I.runs[r].gid_base = static_cast<uint32_t>(N);
      N += I.kv[r].n;
      max_ikey = std::max(max_ikey, I.kv[r].max_klen);
    }
    if (N >= (1ull << 32)) return Fail(YBGPU_NOT_SUPPORTED, "more than 2^32 entries in one job: shard the compaction");
    if (max_ikey > 1008 + 8) return Fail(YBGPU_NOT_SUPPORTED, "user keys longer than 1008 bytes are not supported");
    Sfinal = std::max(32, N ? static_cast<int>(((std::max<uint32_t>(max_ikey, 8) - 8 + 16) + 15) & ~15u) : 32);
    CUDA_TRY(end_phase());
    for (int r = 0; r < k; r++) {
      RunView& rv = I.runs[r];
      CUDA_TRY(DevAlloc(&I.mem, &rv.rec, static_cast<size_t>(rv.n_entries) * Sfinal + 16));
      CUDA_TRY(DevAlloc(&I.mem, &rv.val_off, static_cast<size_t>(rv.n_entries) + 1));
      CUDA_TRY(DevAlloc(&I.mem, &rv.val_crc, static_cast<size_t>(rv.n_entries) + 1));
      if (rv.n_entries) {
        k_records_from_kv<<<GridFor(rv.n_entries, 256, sms), 256, 0, I.stream>>>(I.kv[r].keys, I.kv[r].koff, I.kv[r].voff, rv.data, rv.n_entries, Sfinal,
                                                                             rv.rec, rv.val_off, I.dJ);
        launches++;
      }
    }
    if (ybgpu_status us = UploadSmall(I.dRuns, I.runs.data(), sizeof(RunView) * k)) return us;
    if (N) { k_value_crc<<<GridFor(N, 256, sms), 256, 0, I.stream>>>(I.dRuns, k, Sfinal); launches++; }
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(end_phase());
    if (ybgpu_status s = CheckDeviceError("kv inputs")) return s;
    ingested = true;
    stats_.path_flags |= YBGPU_PATH_KV_INPUT;
  }
  // ---- probe: restart counts (entry upper bounds), restart interval, key length sample, compression types
  bool verify_pending = opt_.verify_checksums != 0;      // false once the stored blocks' checksums have been verified
  if (blk_base[k] > 0) {
    for (int pass = 0; pass < 2; pass++) {
      k_restart_probe<<<GridFor(blk_base[k], 256, sms), 256, 0, I.stream>>>(I.dRuns, d_blk_base, k, I.dJ);
      launches++;
      CUDA_TRY(cudaGetLastError());
      if (ybgpu_status s = CheckDeviceError("block scan")) return s;
      if (!I.hJ.n_compressed) break;
      if (pass == 1) return Fail(YBGPU_CORRUPTION, "compressed blocks after decompression");
      // ---- Snappy- (production default, docdb_rocksdb_util.cc:184) and LZ4-compressed data blocks: checksum of the STORED
      // bytes first (format.cc:352-395), then one uncompressed image of all inputs, whatever the codec mix (format.cc:441-500)
      if (verify_pending) {
        for (int r = 0; r < k; r++) {
          RunView& rv = I.runs[r];
          if (!rv.nb) continue;
          k_crc_blocks<<<GridFor(static_cast<uint64_t>(rv.nb) * 32, 256, sms), 256, 0, I.stream>>>(
              const_cast<uint8_t*>(rv.data), reinterpret_cast<const unsigned long long*>(rv.blk_off), rv.blk_size, nullptr, rv.nb, 1, I.dJ);
          launches++;
        }
        verify_pending = false;
      }
      SnapView sv{};
      sv.runs = I.dRuns; sv.blk_base = d_blk_base; sv.k = k;
      CUDA_TRY(DevAlloc(&I.mem, &sv.out_off, static_cast<size_t>(blk_base[k]) + 1));
      CUDA_TRY(DevAlloc(&I.mem, &sv.usize, static_cast<size_t>(blk_base[k])));
      unsigned long long* d_img = nullptr;
      CUDA_TRY(DevAlloc(&I.mem, &d_img, 1));
      k_snappy_sizes<<<GridFor(blk_base[k], 256, sms), 256, 0, I.stream>>>(sv, I.dJ);
      k_scan_u64_single<<<1, 1024, 0, I.stream>>>(sv.out_off, blk_base[k], d_img);
      launches += 2;
      CUDA_TRY(cudaGetLastError());
      if (ybgpu_status s = CheckDeviceError("uncompressed sizes")) return s;
      unsigned long long img_bytes = 0;
      if (ybgpu_status s = ReadSmall(&img_bytes, d_img, 8)) return s;
      uint8_t* img = nullptr;
      CUDA_TRY(DevAlloc(&I.mem, &img, img_bytes + 96));
      CUDA_TRY(cudaMemsetAsync(img, 0, 16, I.stream));
      CUDA_TRY(cudaMemsetAsync(img + 16 + img_bytes, 0, 64, I.stream));
      sv.out = img + 16;
      k_snappy_decode<<<sms * 8, 128, 0, I.stream>>>(sv, I.dJ);
      launches++;
      CUDA_TRY(cudaGetLastError());
      for (int r = 0; r < k; r++) {
        RunView& rv = I.runs[r];
        rv.data = img + 16;
        rv.blk_off = reinterpret_cast<const uint64_t*>(sv.out_off) + blk_base[r];
        rv.blk_size = sv.usize + blk_base[r];
      }
      if (ybgpu_status us = UploadSmall(I.dRuns, I.runs.data(), sizeof(RunView) * k)) return us;
      // the probe starts over on the uncompressed image
      CUDA_TRY(cudaMemsetAsync(&I.dJ->n_compressed, 0, 2 * sizeof(uint32_t), I.stream));   // n_compressed, n_lz4
      CUDA_TRY(cudaMemsetAsync(I.dJ->restart_interval, 0, sizeof(uint32_t) * MAX_RUNS, I.stream));
      CUDA_TRY(cudaMemsetAsync(&I.dJ->max_ikey_len, 0, sizeof(uint32_t), I.stream));
      if (I.hJ.n_compressed > I.hJ.n_lz4) stats_.path_flags |= YBGPU_PATH_SNAPPY;
      if (I.hJ.n_lz4) stats_.path_flags |= YBGPU_PATH_LZ4;
      tick("uncompress");
    }
    CUDA_TRY(end_phase());
    if (shutdown()) return Fail(YBGPU_SHUTDOWN_IN_PROGRESS, "Database shutdown or Column family drop during compaction");
  }
  if (try_ingest) {
    // exact entry counts: (restarts - 1) x restart interval + the last interval (probe), scanned per file
    k_block_counts<<<GridFor(blk_base[k], 256, sms), 256, 0, I.stream>>>(I.dRuns, d_blk_base, k, I.dJ);
    k_scan_blk_counts<<<k, 1024, 0, I.stream>>>(I.dRuns, d_totals);
    launches += 2;
    CUDA_TRY(cudaGetLastError());
    std::vector<uint32_t> cap(k + 1, 0);
    if (ybgpu_status s = ReadSmall(cap.data(), d_totals, 4 * static_cast<size_t>(k))) return s;
    {
      uint64_t cap_total = 0;
      for (int r = 0; r < k; r++) cap_total += cap[r];
      if (cap_total >= (1ull << 32)) return Fail(YBGPU_NOT_SUPPORTED, "more than 2^32 entries in one job: shard the compaction");
    }
    // record stride: user key + 16-byte trailer, from the longest key the probe's sample met; a longer key inside
    // k_ingest costs one more attempt with the widest stride the kernel takes (64-byte internal keys)
    const int S_widest = 16 * ING_NVI + 16;
    const uint32_t sample_max = std::max<uint32_t>(I.hJ.max_ikey_len, 8);
    Sfinal = std::min(S_widest, std::max(32, static_cast<int>(((sample_max - 8 + 16) + 15) & ~15u)));
    IngestView iv{};
    CUDA_TRY(DevAlloc(&I.mem, &iv.ticket, 1));
    CUDA_TRY(cudaFuncSetAttribute(k_ingest, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(ING_SMEM)));
    for (int attempt = 0; attempt < 2; attempt++) {
      for (int r = 0; r < k; r++) {
        RunView& rv = I.runs[r];
        CUDA_TRY(DevAlloc(&I.mem, &rv.rec, static_cast<size_t>(cap[r]) * Sfinal + 16));
        if (attempt == 0) {
          CUDA_TRY(DevAlloc(&I.mem, &rv.val_off, static_cast<size_t>(cap[r]) + 1));
          CUDA_TRY(DevAlloc(&I.mem, &rv.val_crc, static_cast<size_t>(cap[r]) + 1));
        }
      }
      if (ybgpu_status us = UploadSmall(I.dRuns, I.runs.data(), sizeof(RunView) * k)) return us;
      CUDA_TRY(cudaMemsetAsync(iv.ticket, 0, 4, I.stream));
      CUDA_TRY(cudaMemsetAsync(&I.dJ->ingest_fallback, 0, sizeof(int), I.stream));
      iv.runs = I.dRuns; iv.blk_base = d_blk_base; iv.totals = d_totals; iv.range = d_range;
      iv.k = k; iv.S = Sfinal; iv.verify = verify_pending ? 1 : 0;
      const int grid = static_cast<int>(std::min<uint64_t>((blk_base[k] + ING_BATCH - 1) / ING_BATCH, static_cast<uint64_t>(sms) * 2));
      k_ingest<<<grid, ING_THREADS, ING_SMEM, I.stream>>>(iv, I.dJ);
      launches++;
      CUDA_TRY(cudaGetLastError());
      if (ybgpu_status s = CheckDeviceError("ingest")) return s;
      if (I.hJ.ingest_fallback != ING_FALLBACK_WIDER || Sfinal == S_widest) break;
      Sfinal = S_widest;
      stats_.path_flags |= YBGPU_PATH_INGEST_RETRY;
    }
    CUDA_TRY(end_phase());
    tick("ingest");
    if (!I.hJ.ingest_fallback) {
      const std::vector<uint32_t>& h_totals = cap;
      for (int r = 0; r < k; r++) {
        I.runs[r].n_entries = h_totals[r];
        I.runs[r].restart_interval = I.hJ.restart_interval[r];
        I.runs[r].gid_base = static_cast<uint32_t>(N);
        N += h_totals[r];
      }
      max_ikey = I.hJ.max_ikey_len;
      ingested = true;
      stats_.path_flags |= YBGPU_PATH_FUSED_INGEST;
    } else {
    }
  }
  if (!ingested) {
    // ---- general path. K1: prepass + scan per file
    phase = 0;                             // "block scan" = everything up to the end of the prepass (probe, a failed fused attempt)
    stats_.path_flags |= YBGPU_PATH_GENERAL_DECODE;
    if (verify_pending) {
      // ReadBlock's checksum verification (table/format.cc:352-395) for every input block
      for (int r = 0; r < k; r++) {
        RunView& rv = I.runs[r];
        if (!rv.nb) continue;
        k_crc_blocks<<<GridFor(static_cast<uint64_t>(rv.nb) * 32, 256, sms), 256, 0, I.stream>>>(
            const_cast<uint8_t*>(rv.data), reinterpret_cast<const unsigned long long*>(rv.blk_off), rv.blk_size, nullptr, rv.nb, 1, I.dJ);
        launches++;
      }
    }
    if (blk_base[k]) {
      k_prepass<<<GridFor(static_cast<uint64_t>(blk_base[k]) * 32, 256, sms), 256, 0, I.stream>>>(I.dRuns, d_blk_base, k, I.dJ);
      launches++;
    }
    if (k) { k_scan_blk_counts<<<k, 1024, 0, I.stream>>>(I.dRuns, d_totals); launches++; }
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(end_phase());
    if (ybgpu_status s = CheckDeviceError("block scan")) return s;
    tick("block scan");
    if (shutdown()) return Fail(YBGPU_SHUTDOWN_IN_PROGRESS, "Database shutdown or Column family drop during compaction");
    std::vector<uint32_t> h_totals(k + 1, 0);
    if (k) { if (ybgpu_status s = ReadSmall(h_totals.data(), d_totals, 4 * static_cast<size_t>(k))) return s; }
    for (int r = 0; r < k; r++) {
      const uint32_t n = h_totals[r];
      I.runs[r].n_entries = n;
      I.runs[r].restart_interval = I.hJ.restart_interval[r];
      if (N + n >= (1ull << 32)) return Fail(YBGPU_NOT_SUPPORTED, "more than 2^32 entries in one job: shard the compaction");
      I.runs[r].gid_base = static_cast<uint32_t>(N);
      N += n;
    }
    max_ikey = I.hJ.max_ikey_len;
    if (max_ikey > 1008 + 8) return Fail(YBGPU_NOT_SUPPORTED, "user keys longer than 1008 bytes are not supported");
    const int S = N ? static_cast<int>(((max_ikey - 8 + 16) + 15) & ~15u) : 32;   // user key + 16-byte trailer
    Sfinal = std::max(S, 32);

    // ---- K1': decode
    std::vector<uint32_t> group_base(k + 1, 0);
    for (int r = 0; r < k; r++) {
      RunView& rv = I.runs[r];
      CUDA_TRY(DevAlloc(&I.mem, &rv.rec, static_cast<size_t>(rv.n_entries) * Sfinal + 16));
      CUDA_TRY(DevAlloc(&I.mem, &rv.val_off, static_cast<size_t>(rv.n_entries) + 1));
      CUDA_TRY(DevAlloc(&I.mem, &rv.val_crc, static_cast<size_t>(rv.n_entries) + 1));
      group_base[r + 1] = group_base[r] + (rv.nb + DEC_WB - 1) / DEC_WB;
    }
    if (ybgpu_status us = UploadSmall(I.dRuns, I.runs.data(), sizeof(RunView) * k)) return us;
    if (group_base[k]) {
      uint32_t* d_group_base = nullptr;
      CUDA_TRY(DevAlloc(&I.mem, &d_group_base, k + 1));
      if (ybgpu_status us = UploadSmall(d_group_base, group_base.data(), 4 * (k + 1))) return us;
      const int grid = GridFor(static_cast<uint64_t>(group_base[k]) * 32, 128, sms);
      // fast path: shared-prefix inputs, internal keys of at most 64 bytes, no HybridTime filter / key range
      bool fast = d_range == nullptr && max_ikey <= 64;
      for (int r = 0; r < k; r++) fast = fast && I.runs[r].key_encoding == 1 && I.runs[r].ht_filter == 0xfffffffffffffffeull && I.runs[r].cf_n == 0;
      if (fast && getenv("YBGPU_NO_FAST_DECODE") == nullptr) {
        stats_.path_flags |= YBGPU_PATH_FAST_DECODE;
        if (max_ikey <= 32) k_decode_fast<2><<<grid, 128, 0, I.stream>>>(I.dRuns, d_group_base, k, Sfinal, I.dJ);
        else if (max_ikey <= 48) k_decode_fast<3><<<grid, 128, 0, I.stream>>>(I.dRuns, d_group_base, k, Sfinal, I.dJ);
        else k_decode_fast<4><<<grid, 128, 0, I.stream>>>(I.dRuns, d_group_base, k, Sfinal, I.dJ);
      } else if (max_ikey <= 128) k_decode_all<128><<<grid, 128, 0, I.stream>>>(I.dRuns, d_group_base, k, Sfinal, d_range, I.dJ);
      else if (max_ikey <= 320) k_decode_all<320><<<grid, 128, 0, I.stream>>>(I.dRuns, d_group_base, k, Sfinal, d_range, I.dJ);
      else k_decode_all<1024><<<grid, 128, 0, I.stream>>>(I.dRuns, d_group_base, k, Sfinal, d_range, I.dJ);
      launches++;
      // per-entry value CRCs for the block encoder (the fused path computes them while verifying)
      if (ybgpu_status us = UploadSmall(I.dRuns, I.runs.data(), sizeof(RunView) * k)) return us;
      k_value_crc<<<GridFor(N, 256, sms), 256, 0, I.stream>>>(I.dRuns, k, Sfinal);
      launches++;
    }
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(end_phase());
  }
  if (ybgpu_status us = UploadSmall(I.dRuns, I.runs.data(), sizeof(RunView) * k)) return us;

  // ---- job parameters
  JobParams hp{};
  hp.S = Sfinal; hp.k = k; hp.bottommost = opt_.bottommost_level; hp.last_sequence = opt_.last_sequence;
  // smem budget: ~74 KB per CTA (records + per-record side arrays) so three CTAs fit one SM
  uint32_t cap = (74u * 1024u - tile_layout::A1 - 64u) / (Sfinal + 8 + tile_layout::RECS_K);
  cap = std::min(cap, 4096u) & ~15u;
  if (cap < 16) return Fail(YBGPU_NOT_SUPPORTED, "record stride too large for a merge tile");
  hp.tile_cap = cap;
  // Target tile size H: the samples of one run are M records apart, so a tile of ordinary data holds about H + M records;
  // only adversarial inputs approach the bound H + 2kM, and the partition is then repeated with a smaller M (below).
  static const uint32_t h_pct = [] { const char* v = getenv("YBGPU_TILE_H_PCT"); const int x = v ? atoi(v) : 0; return static_cast<uint32_t>(x >= 25 && x <= 90 ? x : 65); }();
  hp.H = std::max(1u, cap * h_pct / 100);
  // between two consecutive candidates lie fewer than M records of every run, so a tile of small rows holds at most H + kM
  hp.M = std::max(1u, std::min(cap / 2, cap - hp.H) / std::max(1, k));
  hp.R.enabled = opt_.retention_enabled;
  hp.R.cutoff_ht = opt_.history_cutoff_ht;
  hp.R.table_ttl_ns = opt_.table_ttl_ns;
  hp.R.cutoff_enc.n = static_cast<uint8_t>(doc_ht_encode(opt_.history_cutoff_ht, 0xffffffffu, hp.R.cutoff_enc.b));
  const uint64_t min_other = opt_.retain_delete_markers_in_major_compaction ? 0 : opt_.other_min_ht;
  hp.R.min_other_enc.n = static_cast<uint8_t>(doc_ht_encode(min_other, 0, hp.R.min_other_enc.b));
  hp.R.ht_min_enc.n = static_cast<uint8_t>(doc_ht_encode(0, 0, hp.R.ht_min_enc.b));
  if (lower_.size() > 255 || upper_.size() > 255) return Fail(YBGPU_NOT_SUPPORTED, "key bounds longer than 255 bytes");
  hp.R.lower_len = static_cast<uint32_t>(lower_.size()); memcpy(hp.R.lower, lower_.data(), lower_.size());
  hp.R.upper_len = static_cast<uint32_t>(upper_.size()); memcpy(hp.R.upper, upper_.data(), upper_.size());
  hp.R.has_cotables_cutoff = opt_.cotables_cutoff_ht != YBGPU_HT_INVALID;
  hp.R.cotables_cutoff_ht = opt_.cotables_cutoff_ht;
  if (hp.R.has_cotables_cutoff) hp.R.cotables_cutoff_enc.n = static_cast<uint8_t>(doc_ht_encode(opt_.cotables_cutoff_ht, 0xffffffffu, hp.R.cotables_cutoff_enc.b));

  // Compaction::GetLargestUserKey: given by the caller or the max over the runs' last records.
  if (!opt_.has_largest_user_key) {
    CUDA_TRY(cudaStreamSynchronize(I.stream));
    std::vector<uint8_t> best; bool any = false;
    std::vector<uint8_t> lastrec(static_cast<size_t>(Sfinal) * k);
    for (int r = 0; r < k; r++) {
      if (!I.runs[r].n_entries) continue;
      CUDA_TRY(cudaMemcpyAsync(lastrec.data() + static_cast<size_t>(r) * Sfinal, I.runs[r].rec + static_cast<size_t>(I.runs[r].n_entries - 1) * Sfinal, Sfinal, cudaMemcpyDeviceToHost, I.stream));
    }
    CUDA_TRY(cudaStreamSynchronize(I.stream));
    for (int r = 0; r < k; r++) {
      if (!I.runs[r].n_entries) continue;
      const uint8_t* tmp = lastrec.data() + static_cast<size_t>(r) * Sfinal;
      uint32_t ulen = rec_ulen(tmp, Sfinal);
      std::vector<uint8_t> key(tmp, tmp + ulen);
      if (!any || std::lexicographical_compare(best.begin(), best.end(), key.begin(), key.end())) { best = key; any = true; }
    }
    largest_ = best;
  }
  if (largest_.size() > sizeof(hp.largest)) return Fail(YBGPU_NOT_SUPPORTED, "largest user key too long");
  hp.largest_len = static_cast<uint32_t>(largest_.size());
  memcpy(hp.largest, largest_.data(), largest_.size());
  if (ybgpu_status us = UploadSmall(I.dP, &hp, sizeof(hp))) return us;
  if (ybgpu_status s = CheckDeviceError("decode")) return s;
  tick("decode");
  if (shutdown()) return Fail(YBGPU_SHUTDOWN_IN_PROGRESS, "Database shutdown or Column family drop during compaction");

  if (N == 0) {
    ran_ = true;
    stats_.gpu_kernel_launches = launches;
    return YBGPU_OK;
  }

  // ---- K2: partition (repeated with a smaller sample stride in the rare case a tile comes out larger than the
  // merge kernel's capacity: see k_sample_pos)
  uint32_t* d_tile_lo = nullptr; unsigned long long* d_tile_rank = nullptr;
  for (int attempt = 0;; attempt++) {
    std::vector<uint32_t> sample_base(k + 1, 0);
    for (int r = 0; r < k; r++) sample_base[r + 1] = sample_base[r] + (I.runs[r].n_entries + hp.M - 1) / hp.M;
    const uint32_t n_samples = sample_base[k];
    if (n_samples >= (1u << 28)) return Fail(YBGPU_NOT_SUPPORTED, "too many partition samples");
    const uint32_t n_buckets = static_cast<uint32_t>(N / hp.H) + 2;
    PartView pv{};
    uint32_t* d_sample_base = nullptr;
    CUDA_TRY(DevAlloc(&I.mem, &d_sample_base, k + 1));
    CUDA_TRY(DevAlloc(&I.mem, &pv.pos, static_cast<size_t>(n_samples) * k));
    CUDA_TRY(DevAlloc(&I.mem, &pv.smode, n_samples));
    CUDA_TRY(DevAlloc(&I.mem, &pv.bucket_min, n_buckets));
    CUDA_TRY(DevAlloc(&I.mem, &d_tile_lo, static_cast<size_t>(n_buckets + 1) * k));
    CUDA_TRY(DevAlloc(&I.mem, &d_tile_rank, n_buckets + 1));
    if (ybgpu_status us = UploadSmall(d_sample_base, sample_base.data(), 4 * (k + 1))) return us;
    CUDA_TRY(cudaMemsetAsync(pv.bucket_min, 0xff, static_cast<size_t>(n_buckets) * 8, I.stream));
    pv.runs = I.dRuns; pv.sample_base = d_sample_base; pv.n_samples = n_samples; pv.n_buckets = n_buckets;
    k_sample_pos<<<GridFor(static_cast<uint64_t>(n_samples) * k, 256, sms), 256, 0, I.stream>>>(pv, I.dP, I.dJ, 0);
    k_sample_pos<<<GridFor(static_cast<uint64_t>(n_samples) * k, 256, sms), 256, 0, I.stream>>>(pv, I.dP, I.dJ, 1);
    k_sample_bucket<<<GridFor(n_samples, 256, sms), 256, 0, I.stream>>>(pv, I.dP);
    {
      const uint32_t tchunks = (n_buckets + TILE_CHUNK - 1) / TILE_CHUNK;
      uint32_t* d_tpart = nullptr; uint32_t* d_ttotal = nullptr;
      CUDA_TRY(DevAlloc(&I.mem, &d_tpart, tchunks + 1)); CUDA_TRY(DevAlloc(&I.mem, &d_ttotal, 1));
      k_bucket_counts<<<tchunks, 256, 0, I.stream>>>(pv, d_tpart);
      k_scan_u32_single<<<1, 1024, 0, I.stream>>>(d_tpart, tchunks, d_ttotal);
      k_build_tiles<<<tchunks, 256, 0, I.stream>>>(pv, I.dP, d_tpart, d_ttotal, d_tile_lo, d_tile_rank, I.dJ);
      k_tile_check<<<GridFor(n_buckets + 1, 256, sms), 256, 0, I.stream>>>(I.dRuns, d_tile_lo, k, I.dJ);
    }
    launches += 7;
    CUDA_TRY(cudaGetLastError());
    if (ybgpu_status s = CheckDeviceError("partition")) return s;
    if (I.hJ.max_tile <= cap) break;
    if (hp.M <= 1 || attempt >= 4)
      return Fail(YBGPU_NOT_SUPPORTED, "record stride and run count too large for a merge tile");
    hp.M = std::max(1u, hp.M / 2);
    stats_.path_flags |= YBGPU_PATH_PARTITION_RETRY;
    if (ybgpu_status us = UploadSmall(I.dP, &hp, sizeof(hp))) return us;
    CUDA_TRY(cudaMemsetAsync(&I.dJ->max_tile, 0, sizeof(uint32_t), I.stream));
  }
  CUDA_TRY(end_phase());
  tick("partition");
  const uint32_t n_tiles = I.hJ.n_tiles;

  // ---- K3: merge + filter
  Desc* d_desc = nullptr; ValueRewrite* d_rw = nullptr;
  const uint32_t rewrite_cap = static_cast<uint32_t>(std::min<uint64_t>(N, 1u << 26));
  CUDA_TRY(DevAlloc(&I.mem, &d_desc, N));
  CUDA_TRY(DevAlloc(&I.mem, &d_rw, rewrite_cap));
  MergeView mv{};
  mv.runs = I.dRuns; mv.tile_lo = d_tile_lo; mv.tile_rank = d_tile_rank; mv.desc = d_desc;
  mv.rewrites = d_rw; mv.rewrite_cap = rewrite_cap; mv.n_tiles = n_tiles;
  uint16_t* d_fk16 = nullptr;
  if (opt_.filter_policy != YBGPU_FILTER_NONE && getenv("YBGPU_NO_FK16") == nullptr) CUDA_TRY(DevAlloc(&I.mem, &d_fk16, N));
  mv.fk16 = d_fk16;
  uint32_t* d_fkh = nullptr;
  if (d_fk16) CUDA_TRY(DevAlloc(&I.mem, &d_fkh, N));
  mv.fkh = d_fkh;
  mv.S = Sfinal; mv.k = k; mv.cap = cap;
  const size_t smem = tile_layout::bytes(Sfinal, cap);
  CUDA_TRY(cudaFuncSetAttribute(k_merge_filter, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  k_merge_filter<<<n_tiles, MERGE_THREADS, smem, I.stream>>>(mv, I.dP, I.dJ);
  launches++;
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(end_phase());
  if (ybgpu_status s = CheckDeviceError("merge")) return s;
  tick("merge");
  if (shutdown()) return Fail(YBGPU_SHUTDOWN_IN_PROGRESS, "Database shutdown or Column family drop during compaction");

  // ---- K4: survivor scan + dense list; K5: block encode
  I.n_out = I.hJ.n_kept; I.out_key_bytes = I.hJ.out_key_bytes; I.out_val_bytes = I.hJ.out_val_bytes;
  const uint32_t n_chunks = static_cast<uint32_t>((N + EMIT_CHUNK - 1) / EMIT_CHUNK);
  Sums3* d_partial = nullptr;
  CUDA_TRY(DevAlloc(&I.mem, &d_partial, n_chunks + 1));
  I.d_desc = d_desc; I.d_partial = d_partial; I.d_rw = d_rw; I.N = N; I.S = Sfinal; I.n_chunks = n_chunks;
  // the chunk sums place survivors among dropped entries: k_compact_desc needs them now, k_emit when the KV stream is asked for
  I.partial_ready = false;
  if (I.n_out != N) { if (ybgpu_status s = EnsureChunkSums()) return s; launches += 2; }
  if (I.n_out >= (1ull << 32)) return Fail(YBGPU_NOT_SUPPORTED, "too many output entries");
  const uint32_t n = static_cast<uint32_t>(I.n_out);
  if (n) {
    const uint32_t ri = static_cast<uint32_t>(opt_.block_restart_interval);
    if (ri == 0 || (ri & (ri - 1)) || ri > 64)
      return Fail(YBGPU_NOT_SUPPORTED, "block_restart_interval must be a power of two <= 64 for the GPU block encoder");
    if (opt_.output_key_encoding != YBGPU_KEY_ENCODING_SHARED_PREFIX && opt_.output_key_encoding != YBGPU_KEY_ENCODING_THREE_SHARED_PARTS)
      return Fail(YBGPU_INVALID_ARGUMENT, "unknown output_key_encoding");
    if (static_cast<uint64_t>(n) == N) {
      I.d_kept = d_desc;                                  // nothing was dropped: the merged-order list IS the survivor list
    } else {
      CUDA_TRY(DevAlloc(&I.mem, &I.d_kept, n));
      k_compact_desc<<<n_chunks, EMIT_THREADS, 0, I.stream>>>(d_desc, N, d_partial, I.d_kept);
    }
    EncView& E = I.enc;
    E.runs = I.dRuns; E.kept = I.d_kept; E.rewrites = d_rw; E.n = n; E.ri = ri;
    E.ri_shift = 0; while ((1u << E.ri_shift) < ri) E.ri_shift++;
    E.key_encoding = opt_.output_key_encoding;
    E.block_size = opt_.block_size; E.deviation = static_cast<uint32_t>(std::max(0, opt_.block_size_deviation));
    {
      const double avg = static_cast<double>(I.out_key_bytes + I.out_val_bytes) / n + 3.0;
      E.guess = static_cast<uint32_t>(std::max(1.0, 0.85 * opt_.block_size / avg));
    }
    CUDA_TRY(DevAlloc(&I.mem, &E.nr, n)); CUDA_TRY(DevAlloc(&I.mem, &E.shared, n)); CUDA_TRY(DevAlloc(&I.mem, &E.D, n));
    CUDA_TRY(DevAlloc(&I.mem, &E.P, static_cast<size_t>(n) + 1)); CUDA_TRY(DevAlloc(&I.mem, &E.QQ, n));
    CUDA_TRY(DevAlloc(&I.mem, &E.next, n)); CUDA_TRY(DevAlloc(&I.mem, &E.exit1, n));
    E.fk_len = nullptr; E.fk_src = nullptr; E.fkh_src = nullptr;
    if (opt_.filter_policy != YBGPU_FILTER_NONE) {
      if (opt_.filter_policy != YBGPU_FILTER_DOCKEY_V3) return Fail(YBGPU_INVALID_ARGUMENT, "unknown filter_policy");
      CUDA_TRY(DevAlloc(&I.mem, &E.fk_len, n));
      E.fk_src = d_fk16;
      E.fkh_src = d_fkh;
    }
    CUDA_TRY(DevAlloc(&I.mem, &E.max_add, 1));
    CUDA_TRY(cudaMemsetAsync(E.max_add, 0, 4, I.stream));
    // ---- block planning: per-entry sizes with the chunk partials of P, QQ and the filter-key ordinals in one pass, one scan
    // launch over all partial arrays, one launch that applies them (encode_kernels.cuh)
    const uint32_t pc = (n + SCAN_CHUNK - 1) / SCAN_CHUNK;
    const uint32_t rows = (n + ri - 1) / ri;
    const uint32_t qchunks = (rows + QROWS - 1) / QROWS;
    unsigned long long *d_pp = nullptr, *d_qp = nullptr;
    uint32_t* d_counts = nullptr;                         // [0] data blocks, [1] distinct filter keys
    uint8_t* d_is_new = nullptr; uint32_t* d_npart = nullptr; uint32_t* d_new_entry = nullptr; uint32_t* d_hash = nullptr;
    CUDA_TRY(DevAlloc(&I.mem, &d_pp, pc + 1));
    CUDA_TRY(DevAlloc(&I.mem, &d_qp, static_cast<size_t>(qchunks) * ri + 1));
    CUDA_TRY(DevAlloc(&I.mem, &d_counts, 2));
    CUDA_TRY(cudaMemsetAsync(d_counts, 0, 8, I.stream));
    host::FilterGeometry hg{};
    if (E.fk_len) {
      hg = host::ComputeFilterGeometry(opt_.filter_block_size ? opt_.filter_block_size : 65536u);
      if (hg.max_keys == 0) return Fail(YBGPU_INVALID_ARGUMENT, "filter_block_size too small");
      CUDA_TRY(DevAlloc(&I.mem, &d_is_new, n)); CUDA_TRY(DevAlloc(&I.mem, &d_npart, pc + 1));
      // no more distinct filter keys than entries: sized before the count is known, so that one pass can fill both
      CUDA_TRY(DevAlloc(&I.mem, &d_new_entry, static_cast<size_t>(n) + 1));
      if (((hg.filter_bytes + 7u) & ~7u) <= FILTER_SMEM_MAX) CUDA_TRY(DevAlloc(&I.mem, &d_hash, n));
    }
    k_plan_entries<<<(n + PLAN_CHUNK - 1) / PLAN_CHUNK, 256, 0, I.stream>>>(E, Sfinal, d_is_new, d_pp, pc, d_qp, qchunks, d_npart);
    k_plan_scan<<<ri + 2, 1024, 0, I.stream>>>(d_pp, pc, d_qp, qchunks, d_npart, d_counts + 1);
    k_plan_final<<<pc + (qchunks * ri + 255) / 256, 256, 0, I.stream>>>(E, Sfinal, d_is_new, d_pp, pc, d_qp, qchunks, d_npart, d_new_entry, d_hash);
    launches += 3;
    // block cuts
    const uint32_t nsegs = (n + SEG - 1) / SEG;
    const uint32_t ngroups = (nsegs + GROUP_SEGS - 1) / GROUP_SEGS;
    uint32_t *d_gexit = nullptr, *d_group_first = nullptr, *d_seg_first = nullptr, *d_seg_blocks = nullptr;
    CUDA_TRY(DevAlloc(&I.mem, &d_gexit, static_cast<size_t>(ngroups) * SEG));
    CUDA_TRY(DevAlloc(&I.mem, &d_group_first, ngroups)); CUDA_TRY(DevAlloc(&I.mem, &d_seg_first, nsegs));
    CUDA_TRY(DevAlloc(&I.mem, &d_seg_blocks, nsegs));
    k_seg_exit<<<nsegs, 256, 0, I.stream>>>(E);
    k_group_exit<<<static_cast<uint32_t>((static_cast<uint64_t>(ngroups) * SEG + 255) / 256), 256, 0, I.stream>>>(E, d_gexit, ngroups);
    k_chain_groups<<<1, 32, 0, I.stream>>>(E, d_gexit, ngroups, d_group_first);
    k_group_fill<<<(ngroups + 127) / 128, 128, 0, I.stream>>>(E, d_group_first, ngroups, d_seg_first, nsegs);
    k_count_starts<<<(nsegs + 127) / 128, 128, 0, I.stream>>>(E, d_seg_first, nsegs, d_seg_blocks);
    k_scan_u32_single<<<1, 1024, 0, I.stream>>>(d_seg_blocks, nsegs, d_counts);
    launches += 6;
    uint32_t counts[2] = {0, 0};
    if (ybgpu_status s = ReadSmall(counts, d_counts, 8)) return s;
    const uint32_t nblocks = counts[0], n_keys = counts[1];
    I.n_blocks = nblocks;
    CUDA_TRY(DevAlloc(&I.mem, &I.d_block_first, static_cast<size_t>(nblocks) + 1));
    CUDA_TRY(DevAlloc(&I.mem, &I.d_block_off, static_cast<size_t>(nblocks) + 1));
    unsigned long long* d_total = nullptr;                // [0] file length, [1] largest block (contents + trailer)
    CUDA_TRY(DevAlloc(&I.mem, &d_total, 2));
    CUDA_TRY(cudaMemsetAsync(d_total, 0, 16, I.stream));
    k_block_fill<<<(nsegs + 127) / 128, 128, 0, I.stream>>>(E, d_seg_first, nsegs, d_seg_blocks, I.d_block_first, I.d_block_off, d_total + 1);
    {
      const uint32_t bc = (nblocks + SCAN_CHUNK - 1) / SCAN_CHUNK;
      unsigned long long* d_bpart = nullptr;
      CUDA_TRY(DevAlloc(&I.mem, &d_bpart, static_cast<size_t>(bc) + 1));
      k_u64_chunk_sums<<<bc, 256, 0, I.stream>>>(I.d_block_off, nblocks, d_bpart);
      k_scan_u64_single<<<1, 1024, 0, I.stream>>>(d_bpart, bc, d_total);
      k_u64_chunk_final<<<bc, 256, 0, I.stream>>>(I.d_block_off, nblocks, d_bpart);
      launches += 4;
    }
    unsigned long long total_and_max[2] = {0, 0};
    if (ybgpu_status s = ReadSmall(total_and_max, d_total, 16)) return s;
    const unsigned long long total = total_and_max[0];
    if (ybgpu_status us = UploadSmall(I.d_block_off + nblocks, &total, 8)) return us;
    I.out_file_len = total;
    CUDA_TRY(DevAlloc(&I.mem, &I.out_file, total + 64));
    {
      const size_t esm = ENC_SMEM_CAP + 32;
      const bool tsp = E.key_encoding == YBGPU_KEY_ENCODING_THREE_SHARED_PARTS;
      const bool v3 = getenv("YBGPU_ENC_V3") != nullptr;           // A/B: the image-CRC assembler of round 1
      // v5 (warp per block, no block image): one scratch row per lane for header + key delta + rewritten value prefix
      const uint32_t G = ((4u + 28u + static_cast<uint32_t>(Sfinal) + 32u + 7u) & ~7u) + 4u;   // bytes; an odd number of words (bank spread)
      const size_t v5_smem = 4096 + static_cast<size_t>(ENC5_THREADS) * G;
      const bool v5 = !v3 && getenv("YBGPU_ENC_V4") == nullptr && v5_smem <= 96 * 1024;
      if (!v3) stats_.path_flags |= YBGPU_PATH_ENCODER_V4;
      CUDA_TRY(cudaEventRecord(I.enc_ev[0], I.stream));
      if (v5) {
        stats_.path_flags |= YBGPU_PATH_ENCODER_V5;
        auto kern = tsp ? k_encode_v5<2> : k_encode_v5<1>;
        CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(v5_smem)));
        static int occ_cache[2][64] = {};
        int& occ = occ_cache[tsp ? 1 : 0][(Sfinal >> 4) & 63];
        if (!occ) {
          CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, ENC5_THREADS, v5_smem));
          if (occ < 1) occ = 1;
        }
        const uint32_t grid = std::min<uint32_t>((nblocks + ENC5_THREADS / 32 - 1) / (ENC5_THREADS / 32), static_cast<uint32_t>(sms) * occ);
        kern<<<grid, ENC5_THREADS, v5_smem, I.stream>>>(E, Sfinal, I.d_block_first, nblocks, I.d_block_off, I.out_file, G);
        launches++;
      } else {
        auto smem_kernel = v3 ? (tsp ? k_encode_smem<2> : k_encode_smem<1>) : (tsp ? k_encode_v4<2> : k_encode_v4<1>);
        auto fused_kernel = tsp ? k_encode_fused<2> : k_encode_fused<1>;
        CUDA_TRY(cudaFuncSetAttribute(smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(esm)));
        smem_kernel<<<std::min<uint32_t>(nblocks, sms * 8), ENC_THREADS, esm, I.stream>>>(E, Sfinal, I.d_block_first, nblocks, I.d_block_off, I.out_file);
        launches++;
        // blocks whose image does not fit shared memory (huge values)
        if (total_and_max[1] > ENC_SMEM_CAP) {
          fused_kernel<<<std::min<uint32_t>(nblocks, sms * 4), ENC_THREADS, 0, I.stream>>>(E, Sfinal, I.d_block_first, nblocks, I.d_block_off, I.out_file, ENC_SMEM_CAP);
          launches++;
          stats_.path_flags |= YBGPU_PATH_ENCODER_FUSED;
        }
      }
      CUDA_TRY(cudaEventRecord(I.enc_ev[1], I.stream));
      I.enc_timed = true;
    }
    const bool lz4_out = opt_.output_compression == YBGPU_COMPRESSION_LZ4;
    if ((opt_.output_compression == YBGPU_COMPRESSION_SNAPPY || lz4_out) && nblocks) {
      // ---- WriteBlock's CompressBlock for every data block (snappy_kernels.cuh, lz4_kernels.cuh): encode into a scratch
      // image, keep what saves 12.5 %, prefix-sum the stored sizes into the final offsets, move the blocks
      SnapCompView C{};
      C.raw = I.out_file; C.raw_off = I.d_block_off; C.nblocks = nblocks;
      unsigned long long* d_foff = nullptr; unsigned long long* d_ftotal = nullptr; unsigned long long* d_fpart = nullptr;
      const uint32_t bc = (nblocks + SCAN_CHUNK - 1) / SCAN_CHUNK;
      CUDA_TRY(DevAlloc(&I.mem, &C.comp, total + 64));
      CUDA_TRY(DevAlloc(&I.mem, &C.csize, nblocks));
      CUDA_TRY(DevAlloc(&I.mem, &d_foff, static_cast<size_t>(nblocks) + 1));
      CUDA_TRY(DevAlloc(&I.mem, &d_ftotal, 1));
      CUDA_TRY(DevAlloc(&I.mem, &d_fpart, static_cast<size_t>(bc) + 1));
      C.fsize = d_foff;
      const uint32_t cgrid = std::min<uint32_t>((nblocks + SNAPC_WARPS - 1) / SNAPC_WARPS, static_cast<uint32_t>(sms) * 4);
      // A/B switch (same binary): how the encoder forms the hash groups of a batch, see snapc_prepare
      const char* sv = getenv("YBGPU_SNAPC_VARIANT");
      const int variant = sv ? atoi(sv) : 0;
      for (auto& e : I.snap_ev) if (!e) CUDA_TRY(cudaEventCreate(&e));
      {
        // 48 KB of static tables per CTA: ask for the largest shared-memory carve-out so that four CTAs share an SM (a hint;
        // without it the driver may settle for a carve-out that holds one)
        static std::once_flag hinted;                      // ranges of a pipelined compaction run on several host threads
        std::call_once(hinted, [] {
          (void)cudaFuncSetAttribute(k_snappy_compress<0>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
          (void)cudaFuncSetAttribute(k_snappy_compress<1>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
          (void)cudaFuncSetAttribute(k_snappy_compress<2>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
          (void)cudaFuncSetAttribute(k_lz4_compress, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
          (void)cudaGetLastError();
        });
      }
      if (trace) {                                         // what the runtime expects to keep resident (4 = the tables' limit)
        int occ = -1;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, lz4_out ? k_lz4_compress : k_snappy_compress<0>, SNAPC_WARPS * 32, 0) != cudaSuccess)
          (void)cudaGetLastError();
        fprintf(stderr, "[ybgpu trace] %s encoder: %u blocks, grid %u x %d threads, variant %d, resident CTAs per SM %d\n", lz4_out ? "lz4" : "snappy",
                nblocks, cgrid, SNAPC_WARPS * 32, lz4_out ? 0 : variant, occ);
      }
      CUDA_TRY(cudaEventRecord(I.snap_ev[0], I.stream));
      if (lz4_out) k_lz4_compress<<<cgrid, SNAPC_WARPS * 32, 0, I.stream>>>(C);
      else if (variant == 2) k_snappy_compress<2><<<cgrid, SNAPC_WARPS * 32, 0, I.stream>>>(C);
      else if (variant == 1) k_snappy_compress<1><<<cgrid, SNAPC_WARPS * 32, 0, I.stream>>>(C);
      else k_snappy_compress<0><<<cgrid, SNAPC_WARPS * 32, 0, I.stream>>>(C);
      CUDA_TRY(cudaEventRecord(I.snap_ev[1], I.stream));
      k_u64_chunk_sums<<<bc, 256, 0, I.stream>>>(d_foff, nblocks, d_fpart);
      k_scan_u64_single<<<1, 1024, 0, I.stream>>>(d_fpart, bc, d_ftotal);
      k_u64_chunk_final<<<bc, 256, 0, I.stream>>>(d_foff, nblocks, d_fpart);
      unsigned long long ftotal = 0;
      if (ybgpu_status s = ReadSmall(&ftotal, d_ftotal, 8)) return s;
      if (ybgpu_status us = UploadSmall(d_foff + nblocks, &ftotal, 8)) return us;
      CUDA_TRY(DevAlloc(&I.mem, &C.out, ftotal + 64));
      CUDA_TRY(cudaEventRecord(I.snap_ev[2], I.stream));
      k_snappy_gather<<<GridFor(static_cast<uint64_t>(nblocks) * 32, 256, sms), 256, 0, I.stream>>>(C);
      CUDA_TRY(cudaEventRecord(I.snap_ev[3], I.stream));
      I.snap_timed = true;
      launches += 5;
      stats_.path_flags |= lz4_out ? YBGPU_PATH_LZ4_OUTPUT : YBGPU_PATH_SNAPPY_OUTPUT;
      // the uncompressed table and the scratch image are done with once the gather has run (stream-ordered frees): the job's
      // footprint stays at one output table for the later phases and for the jobs running beside this one
      for (void* dead : {static_cast<void*>(I.out_file), static_cast<void*>(C.comp)}) CUDA_TRY(I.mem.Free(dead, I.stream));
      I.out_file = C.out; I.out_file_len = ftotal; I.d_block_off = d_foff;
    }
    if (E.fk_len) {
      // ---- bloom filter blocks: distinct filter keys -> ordinals -> 64 KB blocks of max_keys keys each
      BloomGeometry g{hg.num_lines, hg.num_probes, hg.max_keys, hg.filter_bytes, (hg.filter_bytes + 7u) & ~7u};
      // a (possibly empty) block is always flushed at Finish (block_based_table_builder.cc:768-770)
      const uint32_t nfb = std::max<uint32_t>(1, (n_keys + g.max_keys - 1) / g.max_keys);
      I.n_filter_blocks = nfb; I.filter_block_bytes = g.block_bytes;
      I.filter_key_stride = static_cast<uint32_t>((max_ikey + 2 + 7) & ~7u);
      CUDA_TRY(DevAlloc(&I.mem, &I.d_filters, static_cast<size_t>(nfb) * g.dev_stride + 16));
      CUDA_TRY(DevAlloc(&I.mem, &I.d_filter_keys, static_cast<size_t>(nfb) * 2 * I.filter_key_stride));
      CUDA_TRY(DevAlloc(&I.mem, &I.d_filter_first, nfb));
      CUDA_TRY(cudaMemsetAsync(I.d_filters, 0, static_cast<size_t>(nfb) * g.dev_stride, I.stream));
      if (n_keys && d_hash) {
        CUDA_TRY(cudaFuncSetAttribute(k_filter_build_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(g.dev_stride)));
        const uint32_t resident = std::max<uint32_t>(1, std::min<uint32_t>(2, (200u * 1024u) / (g.dev_stride + 1024u))) * sms;   // CTAs that fit at once
        const uint32_t parts = std::max<uint32_t>(1, std::min<uint32_t>(8, resident / nfb));
        k_filter_build_smem<<<std::min<uint32_t>(nfb * parts, resident * 4), 1024, g.dev_stride, I.stream>>>(d_hash, n_keys, g, nfb, parts, I.d_filters);
      } else if (n_keys) {
        k_filter_build<<<GridFor(n_keys, 256, sms), 256, 0, I.stream>>>(E, Sfinal, d_new_entry, n_keys, g, I.d_filters);
      }
      k_filter_finish<<<GridFor(static_cast<uint64_t>(nfb) * 2, 256, sms), 256, 0, I.stream>>>(E, Sfinal, d_new_entry, n_keys, g, nfb, I.d_filters,
                                                                                              I.d_filter_keys, I.filter_key_stride, I.d_filter_first);
      launches += 1 + (n_keys ? 1 : 0);
    }
    if (opt_.compute_user_boundary_values && opt_.retention_enabled) {
      const int bgrid = static_cast<int>(std::max<uint64_t>(1, std::min<uint64_t>((n + 255) / 256, static_cast<uint64_t>(sms) * 2)));
      BvCand* d_cand = nullptr;
      CUDA_TRY(DevAlloc(&I.mem, &d_cand, static_cast<size_t>(bgrid) * 2 * BV_MAXC));
      CUDA_TRY(DevAlloc(&I.mem, &I.d_bv, 1));
      CUDA_TRY(cudaMemsetAsync(d_cand, 0, sizeof(BvCand) * static_cast<size_t>(bgrid) * 2 * BV_MAXC, I.stream));
      CUDA_TRY(cudaMemsetAsync(I.d_bv, 0, sizeof(BvOut), I.stream));
      k_boundary_values<<<bgrid, 256, 0, I.stream>>>(E, Sfinal, d_cand, I.d_bv);
      k_boundary_values_finish<<<1, 64, 0, I.stream>>>(d_cand, static_cast<uint32_t>(bgrid), I.d_bv);
      launches += 2;
    }
    I.boundary_stride = static_cast<uint32_t>((max_ikey + 2 + 7) & ~7u);
    // slot 2*nblocks (one past the per-block pairs): the first key of the file (FileMetaData::smallest)
    CUDA_TRY(DevAlloc(&I.mem, &I.d_boundary, (static_cast<size_t>(nblocks) * 2 + 1) * I.boundary_stride));
    k_boundary_keys<<<GridFor(static_cast<uint64_t>(nblocks) * 2 + 1, 256, sms), 256, 0, I.stream>>>(E, Sfinal, I.d_block_first, nblocks, I.d_boundary, I.boundary_stride);
    launches++;
  }
  CUDA_TRY(end_phase());
  CUDA_TRY(cudaEventRecord(I.ev1, I.stream));
  CUDA_TRY(cudaGetLastError());
  if (ybgpu_status s = CheckDeviceError("encode")) return s;
  tick("encode");
  float ms = 0;
  CUDA_TRY(cudaEventElapsedTime(&ms, I.ev0, I.ev1));
  for (int ph = 0; ph < phase; ph++) {
    float pms = 0;
    CUDA_TRY(cudaEventElapsedTime(&pms, ph ? I.phase_ev[ph - 1] : I.ev0, I.phase_ev[ph]));
    stats_.phase_seconds[ph] = pms / 1e3;
    stats_.phase_launches[ph] = phase_launch_mark[ph] - (ph ? phase_launch_mark[ph - 1] : 0);
  }
  if (I.snap_timed) {                                    // slots 6, 7: k_snappy_compress or k_lz4_compress, k_snappy_gather (one launch each)
    float cms = 0, gms = 0;
    CUDA_TRY(cudaEventElapsedTime(&cms, I.snap_ev[0], I.snap_ev[1]));
    CUDA_TRY(cudaEventElapsedTime(&gms, I.snap_ev[2], I.snap_ev[3]));
    stats_.phase_seconds[6] = cms / 1e3; stats_.phase_launches[6] = 1;
    stats_.phase_seconds[7] = gms / 1e3; stats_.phase_launches[7] = 1;
  }
  if (I.enc_timed) {                                     // slot 5: k_encode_smem alone (one launch)
    float ems = 0;
    CUDA_TRY(cudaEventElapsedTime(&ems, I.enc_ev[0], I.enc_ev[1]));
    stats_.phase_seconds[5] = ems / 1e3; stats_.phase_launches[5] = 1;
  }

  stats_.tiles_inside_rows = I.hJ.n_cont_tiles;
  stats_.num_input_records = I.hJ.n_counted;
  stats_.num_output_records = I.hJ.n_kept;
  stats_.num_record_drop_hidden = I.hJ.n_hidden;
  stats_.num_record_drop_obsolete = I.hJ.n_obsolete;
  stats_.num_record_drop_feed = I.hJ.n_feed_dropped;
  stats_.total_input_raw_key_bytes = I.hJ.in_key_bytes;
  stats_.total_input_raw_value_bytes = I.hJ.in_val_bytes;
  stats_.total_output_raw_key_bytes = I.hJ.out_key_bytes;
  stats_.total_output_raw_value_bytes = I.hJ.out_val_bytes;
  stats_.smallest_seqno = I.hJ.n_kept ? I.hJ.min_seq : 0;
  stats_.largest_seqno = I.hJ.max_seq;
  stats_.num_output_data_blocks = I.n_blocks;
  stats_.output_data_file_size = I.out_file_len;
  stats_.gpu_seconds = ms / 1e3;
  stats_.gpu_kernel_launches = launches + I.readback_launches;
  record_stride_ = Sfinal; num_tiles_ = n_tiles;
  ran_ = true;
  return YBGPU_OK;
}

ybgpu_status Engine::KvStreamSizes(uint64_t* n, uint64_t* kb, uint64_t* vb) const {
  if (!ran_) return const_cast<Engine*>(this)->Fail(YBGPU_ILLEGAL_STATE, "job has not run");
  *n = impl_->n_out; *kb = impl_->out_key_bytes; *vb = impl_->out_val_bytes;
  return YBGPU_OK;
}

// Exclusive chunk sums (survivors, key bytes, value bytes) of the merged-order descriptors: two launches on the job's stream.
ybgpu_status Engine::EnsureChunkSums() {
  Impl& I = *impl_;
  k_emit_sums<<<I.n_chunks, EMIT_THREADS, 0, I.stream>>>(I.d_desc, I.N, I.d_partial);
  k_scan_sums<<<1, 1024, 0, I.stream>>>(I.d_partial, I.n_chunks);
  I.partial_ready = true;
  CUDA_TRY(cudaGetLastError());
  return YBGPU_OK;
}

// The flat KV stream (what CompactionFeed::Feed consumers want) is materialised on demand.
ybgpu_status Engine::EnsureKvStream() {
  Impl& I = *impl_;
  if (I.kv_emitted) return YBGPU_OK;
  CUDA_TRY(cudaSetDevice(opt_.device));
  g_alloc_stream = I.stream;
  CUDA_TRY(DevAlloc(&I.mem, &I.out_keys, I.out_key_bytes + 16));
  CUDA_TRY(DevAlloc(&I.mem, &I.out_vals, I.out_val_bytes + 16));
  CUDA_TRY(DevAlloc(&I.mem, &I.out_koff, I.n_out + 1));
  CUDA_TRY(DevAlloc(&I.mem, &I.out_voff, I.n_out + 1));
  if (I.N) {
    if (!I.partial_ready) { if (ybgpu_status s = EnsureChunkSums()) return s; stats_.gpu_kernel_launches += 2; }
    EmitView ev{};
    ev.runs = I.dRuns; ev.desc = I.d_desc; ev.partial = I.d_partial; ev.rewrites = I.d_rw;
    ev.out_keys = I.out_keys; ev.out_koff = I.out_koff; ev.out_vals = I.out_vals; ev.out_voff = I.out_voff; ev.N = I.N;
    k_emit<<<I.n_chunks, EMIT_THREADS, 0, I.stream>>>(ev, I.S, I.dJ);
    stats_.gpu_kernel_launches++;
  }
  CUDA_TRY(cudaMemcpyAsync(I.out_koff + I.n_out, &I.out_key_bytes, 8, cudaMemcpyHostToDevice, I.stream));
  CUDA_TRY(cudaMemcpyAsync(I.out_voff + I.n_out, &I.out_val_bytes, 8, cudaMemcpyHostToDevice, I.stream));
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaStreamSynchronize(I.stream));
  I.kv_emitted = true;
  return YBGPU_OK;
}

ybgpu_status Engine::FetchKvStream(uint8_t* keys, uint64_t* koff, uint8_t* vals, uint64_t* voff) {
  if (!ran_) return Fail(YBGPU_ILLEGAL_STATE, "job has not run");
  if (ybgpu_status s = EnsureKvStream()) return s;
  Impl& I = *impl_;
  if (I.out_key_bytes) CUDA_TRY(cudaMemcpyAsync(keys, I.out_keys, I.out_key_bytes, cudaMemcpyDeviceToHost, I.stream));
  if (I.out_val_bytes) CUDA_TRY(cudaMemcpyAsync(vals, I.out_vals, I.out_val_bytes, cudaMemcpyDeviceToHost, I.stream));
  CUDA_TRY(cudaMemcpyAsync(koff, I.out_koff, (I.n_out + 1) * 8, cudaMemcpyDeviceToHost, I.stream));
  CUDA_TRY(cudaMemcpyAsync(voff, I.out_voff, (I.n_out + 1) * 8, cudaMemcpyDeviceToHost, I.stream));
  CUDA_TRY(cudaStreamSynchronize(I.stream));
  stats_.d2h_bytes += I.out_key_bytes + I.out_val_bytes + (I.n_out + 1) * 16;
  return YBGPU_OK;
}

// Finished data file (<n>.sst.sblock.0) + what the host needs to write <n>.sst.
ybgpu_status Engine::OutputInfo(uint64_t* data_len, uint32_t* n_blocks, uint32_t* boundary_stride) const {
  if (!ran_) return const_cast<Engine*>(this)->Fail(YBGPU_ILLEGAL_STATE, "job has not run");
  *data_len = impl_->out_file_len; *n_blocks = impl_->n_blocks; *boundary_stride = impl_->boundary_stride;
  return YBGPU_OK;
}

ybgpu_status Engine::FetchOutput(uint8_t* data_file, uint64_t* block_off /*n_blocks+1*/, uint8_t* boundary /*2*n_blocks*stride*/) {
  if (!ran_) return Fail(YBGPU_ILLEGAL_STATE, "job has not run");
  Impl& I = *impl_;
  CUDA_TRY(cudaSetDevice(opt_.device));
  if (I.out_file_len && data_file) CUDA_TRY(cudaMemcpyAsync(data_file, I.out_file, I.out_file_len, cudaMemcpyDeviceToHost, I.stream));
  if (I.n_blocks) {
    if (block_off) { const size_t nb8 = (static_cast<size_t>(I.n_blocks) + 1) * 8; if (ybgpu_status rs = ReadViaMapped(block_off, I.d_block_off, nb8, nb8, 1)) return rs; }
    if (boundary) { const size_t bb = static_cast<size_t>(I.boundary_stride) * 2; if (ybgpu_status rs = ReadViaMapped(boundary, I.d_boundary, bb, bb, I.n_blocks)) return rs; }
  }
  CUDA_TRY(cudaStreamSynchronize(I.stream));
  stats_.d2h_bytes += (data_file ? I.out_file_len : 0) + (block_off ? (static_cast<size_t>(I.n_blocks) + 1) * 8 : 0) +
                      (boundary ? static_cast<size_t>(I.n_blocks) * 2 * I.boundary_stride : 0);
  return YBGPU_OK;
}

ybgpu_status Engine::BeginFetchDataFile(uint8_t* data_file) {
  if (!ran_) return Fail(YBGPU_ILLEGAL_STATE, "job has not run");
  Impl& I = *impl_;
  if (!I.out_file_len) return YBGPU_OK;
  CUDA_TRY(cudaSetDevice(opt_.device));
  if (!I.copy_stream) {
    CUDA_TRY(cudaStreamCreateWithFlags(&I.copy_stream, cudaStreamNonBlocking));
    CUDA_TRY(cudaEventCreateWithFlags(&I.copy_ev, cudaEventDisableTiming));
  }
  CUDA_TRY(cudaEventRecord(I.copy_ev, I.stream));
  CUDA_TRY(cudaStreamWaitEvent(I.copy_stream, I.copy_ev, 0));
  CUDA_TRY(ChunkedCopyAsync(data_file, I.out_file, I.out_file_len, cudaMemcpyDeviceToHost, I.copy_stream));
  I.copy_pending = true;
  return YBGPU_OK;
}

ybgpu_status Engine::EndFetchDataFile() {
  Impl& I = *impl_;
  if (!I.copy_pending) return YBGPU_OK;
  I.copy_pending = false;
  CUDA_TRY(cudaStreamSynchronize(I.copy_stream));
  stats_.d2h_bytes += I.out_file_len;
  return YBGPU_OK;
}

uint64_t Engine::kept_deletions() const { return impl_->hJ.n_kept_deletions; }

// FileMetaData::smallest / largest of the output (db/version_edit.h:101-165): records of
// [u16 key length][internal key], boundary_stride bytes each (zero length: no output).
ybgpu_status Engine::FetchFileBoundaries(uint8_t* smallest, uint8_t* largest) {
  if (!ran_) return Fail(YBGPU_ILLEGAL_STATE, "job has not run");
  Impl& I = *impl_;
  smallest[0] = smallest[1] = 0; largest[0] = largest[1] = 0;
  if (!I.n_blocks) return YBGPU_OK;
  CUDA_TRY(cudaSetDevice(opt_.device));
  if (ybgpu_status rs = ReadViaMapped(smallest, I.d_boundary + static_cast<size_t>(I.n_blocks) * 2 * I.boundary_stride, I.boundary_stride, I.boundary_stride, 1)) return rs;
  if (ybgpu_status rs = ReadViaMapped(largest, I.d_boundary + static_cast<size_t>(I.n_blocks - 1) * 2 * I.boundary_stride, I.boundary_stride, I.boundary_stride, 1)) return rs;
  stats_.d2h_bytes += 2ull * I.boundary_stride;
  return YBGPU_OK;
}

ybgpu_status Engine::FetchUserValues(ybgpu_user_value* smallest, ybgpu_user_value* largest, uint32_t cap, uint32_t* n) {
  if (!ran_) return Fail(YBGPU_ILLEGAL_STATE, "job has not run");
  if (!opt_.compute_user_boundary_values) return Fail(YBGPU_ILLEGAL_STATE, "options.compute_user_boundary_values was not set");
  Impl& I = *impl_;
  *n = 0;
  if (!I.d_bv) return YBGPU_OK;                           // nothing survived / plain RocksDB mode
  CUDA_TRY(cudaSetDevice(opt_.device));
  std::vector<uint8_t> buf(sizeof(BvOut));
  if (ybgpu_status rs = ReadViaMapped(buf.data(), I.d_bv, sizeof(BvOut), sizeof(BvOut), 1)) return rs;
  stats_.d2h_bytes += sizeof(BvOut);
  const BvOut& o = *reinterpret_cast<const BvOut*>(buf.data());
  if (o.overflow) return Fail(YBGPU_NOT_SUPPORTED, "more than 16 range components or a component longer than 255 bytes: boundary values not computed");
  uint32_t m = 0;
  for (uint32_t c = 0; c < o.n_comps && c < BV_MAXC; c++) {
    if (!o.len[0][c] && !o.len[1][c]) continue;
    if (m >= cap) return Fail(YBGPU_INVALID_ARGUMENT, "user value buffers too small");
    smallest[m].tag = largest[m].tag = 10 + c;           // TagForRangeComponent (doc_boundary_values_extractor.cc:108-110)
    smallest[m].len = o.len[0][c]; largest[m].len = o.len[1][c];
    memcpy(smallest[m].value, o.val[0][c], o.len[0][c]);
    memcpy(largest[m].value, o.val[1][c], o.len[1][c]);
    m++;
  }
  *n = m;
  return YBGPU_OK;
}

ybgpu_status Engine::FilterInfo(uint32_t* n_filter_blocks, uint32_t* block_bytes, uint32_t* key_stride) const {
  if (!ran_) return const_cast<Engine*>(this)->Fail(YBGPU_ILLEGAL_STATE, "job has not run");
  *n_filter_blocks = impl_->n_filter_blocks; *block_bytes = impl_->filter_block_bytes; *key_stride = impl_->filter_key_stride;
  return YBGPU_OK;
}

ybgpu_status Engine::FetchFilter(uint8_t* filters, uint8_t* keys, uint32_t* first_entry, uint32_t* block_first) {
  if (!ran_) return Fail(YBGPU_ILLEGAL_STATE, "job has not run");
  Impl& I = *impl_;
  CUDA_TRY(cudaSetDevice(opt_.device));
  const size_t fb = static_cast<size_t>(I.n_filter_blocks) * I.filter_block_bytes, kb = static_cast<size_t>(I.n_filter_blocks) * 2 * I.filter_key_stride;
  if (I.n_filter_blocks) {
    if (ybgpu_status rs = ReadViaMapped(filters, I.d_filters, I.filter_block_bytes, (I.filter_block_bytes + 7u) & ~7u, I.n_filter_blocks)) return rs;
    if (ybgpu_status rs = ReadViaMapped(keys, I.d_filter_keys, kb, kb, 1)) return rs;
    const size_t fe = static_cast<size_t>(I.n_filter_blocks) * 4;
    if (ybgpu_status rs = ReadViaMapped(first_entry, I.d_filter_first, fe, fe, 1)) return rs;
  }
  if (I.n_blocks) { const size_t bf = static_cast<size_t>(I.n_blocks) * 4; if (ybgpu_status rs = ReadViaMapped(block_first, I.d_block_first, bf, bf, 1)) return rs; }
  stats_.d2h_bytes += fb + kb + static_cast<size_t>(I.n_filter_blocks) * 4 + static_cast<size_t>(I.n_blocks) * 4;
  return YBGPU_OK;
}

ybgpu_status Engine::Digest(uint64_t* digest) {
  if (!ran_) return Fail(YBGPU_ILLEGAL_STATE, "job has not run");
  if (ybgpu_status s = EnsureKvStream()) return s;
  Impl& I = *impl_;
  CUDA_TRY(cudaSetDevice(opt_.device));
  int sms = 0;
  CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, opt_.device));
  CUDA_TRY(cudaMemsetAsync(&I.dJ->digest, 0, 8, I.stream));
  if (I.n_out) k_digest<<<GridFor(I.n_out, 256, sms), 256, 0, I.stream>>>(I.out_keys, I.out_koff, I.out_vals, I.out_voff, I.n_out, I.dJ);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(&I.hJ, I.dJ, sizeof(JobDev), cudaMemcpyDeviceToHost, I.stream));
  CUDA_TRY(cudaStreamSynchronize(I.stream));
  *digest = I.hJ.digest;
  return YBGPU_OK;
}

// =============================================================================================
// V: output check (verify_kernels.cuh)
// =============================================================================================
namespace {
// Temporaries of one check, from the stream-ordered pool; returned to it when the check ends, however it ends.
struct VerifyScratch {
  JobMemory& mem;
  cudaStream_t stream;
  std::vector<void*> ptrs;
  VerifyScratch(JobMemory& m, cudaStream_t s) : mem(m), stream(s) {}
  ~VerifyScratch() { for (void* p : ptrs) mem.Free(p, stream); }
  template <typename T>
  cudaError_t Alloc(T** out, size_t count) {
    void* p = nullptr;
    cudaError_t e = mem.Alloc(&p, JobMemory::Padded(count * sizeof(T)), stream);
    if (e == cudaSuccess) { ptrs.push_back(p); *out = reinterpret_cast<T*>(p); }
    return e;
  }
};
const char* VerifyKindName(uint32_t kind) {
  switch (kind) {
    case VERIFY_CHECKSUM: return "block checksum mismatch";
    case VERIFY_COMPRESSED: return "compressed block does not decode";
    case VERIFY_PARSE: return "entry does not parse";
    case VERIFY_ORDER: return "keys out of order";
    case VERIFY_COUNT: return "entry count differs from the merge result";
    case VERIFY_CONTENTS: return "entry differs from the merge result";
    case VERIFY_KEY_TOO_LONG: return "internal key longer than 1016 bytes";
    default: return "unknown failure";
  }
}
}  // namespace

// The table at `file`: nb blocks at d_off (nb + 1 offsets back to back when d_size is null, else with the contents sizes
// d_size). job: also against the merge result of this engine's run.
ybgpu_status Engine::VerifyTable(const uint8_t* file, uint64_t file_len, const unsigned long long* d_off, const uint32_t* d_size,
                                 uint32_t nb, int key_encoding, bool job, ybgpu_output_check* result) {
  Impl& I = *impl_;
  memset(result, 0, sizeof(*result));
  if (nb == 0) return YBGPU_OK;                            // no table was written (compaction_job.cc:950-952)
  int sms = 0;
  CUDA_TRY(EnsureDeviceTables(opt_.device, I.stream, &sms));
  VerifyScratch T(I.mem, I.stream);
  cudaEvent_t ev[2] = {};
  for (auto& e : ev) CUDA_TRY(cudaEventCreate(&e));
  struct EvGuard { cudaEvent_t* e; ~EvGuard() { cudaEventDestroy(e[0]); cudaEventDestroy(e[1]); } } ev_guard{ev};
  JobDev* dV = nullptr;
  uint32_t* d_sz = nullptr;
  CUDA_TRY(T.Alloc(&dV, 1));
  CUDA_TRY(T.Alloc(&d_sz, nb));
  JobDev hV{}; hV.verify_fail = ~0ull;
  CUDA_TRY(cudaEventRecord(ev[0], I.stream));
  if (ybgpu_status us = UploadSmall(dV, &hV, sizeof(hV))) return us;
  k_verify_sizes<<<GridFor(nb, 256, sms), 256, 0, I.stream>>>(file, d_off, d_size, nb, d_sz, dV);
  k_crc_blocks<<<GridFor(static_cast<uint64_t>(nb) * 32, 256, sms), 256, 0, I.stream>>>(const_cast<uint8_t*>(file), d_off, d_sz, nullptr, nb, 2, dV);
  CUDA_TRY(cudaGetLastError());
  if (ybgpu_status s = ReadSmall(&hV, dV, sizeof(JobDev))) return s;
  result->blocks_checked = nb;
  result->blocks_compressed = hV.n_compressed;
  result->bytes_read = file_len;

  VerifyView V{};
  V.data = file; V.off = d_off; V.size = d_sz; V.nblocks = nb; V.key_encoding = key_encoding;
  if (hV.n_compressed) {
    // ---- what ReadBlock would hand to BlockIter: one uncompressed image of the table (UncompressBlockContents,
    // table/format.cc:441-500), by the kernels that uncompress input tables
    RunView rv{};
    rv.data = file; rv.blk_off = reinterpret_cast<const uint64_t*>(d_off); rv.blk_size = d_sz; rv.nb = nb;
    const uint32_t base[2] = {0, nb};
    RunView* d_run = nullptr; uint32_t* d_base = nullptr; unsigned long long* d_img = nullptr;
    SnapView sv{};
    CUDA_TRY(T.Alloc(&d_run, 1)); CUDA_TRY(T.Alloc(&d_base, 2)); CUDA_TRY(T.Alloc(&d_img, 1));
    CUDA_TRY(T.Alloc(&sv.out_off, static_cast<size_t>(nb) + 1)); CUDA_TRY(T.Alloc(&sv.usize, nb));
    if (ybgpu_status us = UploadSmall(d_run, &rv, sizeof(rv))) return us;
    if (ybgpu_status us = UploadSmall(d_base, base, sizeof(base))) return us;
    sv.runs = d_run; sv.blk_base = d_base; sv.k = 1;
    k_snappy_sizes<<<GridFor(nb, 256, sms), 256, 0, I.stream>>>(sv, dV);
    k_scan_u64_single<<<1, 1024, 0, I.stream>>>(sv.out_off, nb, d_img);
    CUDA_TRY(cudaGetLastError());
    unsigned long long img_bytes = 0;
    if (ybgpu_status s = ReadSmall(&img_bytes, d_img, 8)) return s;
    if (ybgpu_status s = ReadSmall(&hV, dV, sizeof(JobDev))) return s;
    // no Snappy or LZ4 stream grows more than 255-fold: a larger announcement is a damaged preamble, not an image to allocate
    if (!hV.error && img_bytes > 256 * file_len + 5ull * nb) { hV.error = DEV_ERR_BAD_BLOCK; hV.error_where = 0; }
    if (!hV.error) {
      uint8_t* img = nullptr;
      CUDA_TRY(T.Alloc(&img, img_bytes + 96));
      CUDA_TRY(cudaMemsetAsync(img, 0, 16, I.stream));
      CUDA_TRY(cudaMemsetAsync(img + 16 + img_bytes, 0, 64, I.stream));
      sv.out = img + 16;
      k_snappy_decode<<<sms * 8, 128, 0, I.stream>>>(sv, dV);
      CUDA_TRY(cudaGetLastError());
      V.data = img + 16; V.off = sv.out_off; V.size = sv.usize;
      result->bytes_read += img_bytes;
    }
  }
  if (!hV.error) {
    V.ri = job ? static_cast<uint32_t>(opt_.block_restart_interval) : 0u;
    V.kcap = job ? I.boundary_stride : VERIFY_MAX_IKEY;
    V.kstride = (V.kcap + 15u) & ~15u;
    auto kern = job ? k_verify_blocks<true> : k_verify_blocks<false>;
    int occ = 0;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, VERIFY_THREADS, 0));
    // a persistent grid: as many warps as stay resident (fewer for a table that came from outside, whose key buffers are sized for the longest key)
    const uint32_t per_sm = static_cast<uint32_t>(std::max(1, job ? occ : std::min(occ, 4)));
    const uint32_t grid = std::min<uint32_t>((nb + VERIFY_THREADS / 32 - 1) / (VERIFY_THREADS / 32), static_cast<uint32_t>(sms) * per_sm);
    CUDA_TRY(T.Alloc(&V.keybuf, static_cast<size_t>(grid) * VERIFY_THREADS * 2 * V.kstride));
    if (job) { V.block_first = I.d_block_first; V.boundary = I.d_boundary; V.boundary_stride = I.boundary_stride; }
    kern<<<grid, VERIFY_THREADS, 0, I.stream>>>(V, job ? I.enc : EncView{}, I.S, dV);
    CUDA_TRY(cudaGetLastError());
  }
  CUDA_TRY(cudaEventRecord(ev[1], I.stream));
  if (ybgpu_status s = ReadSmall(&hV, dV, sizeof(JobDev))) return s;
  float ms = 0;
  CUDA_TRY(cudaEventElapsedTime(&ms, ev[0], ev[1]));
  result->gpu_seconds = ms / 1e3;
  result->entries_parsed = hV.n_counted;
  if (job) result->bytes_read += I.out_val_bytes + static_cast<uint64_t>(I.n_out) * I.S;

  unsigned long long fail = hV.verify_fail;
  if (hV.error == DEV_ERR_COMPRESSED) {
    char buf[160];
    snprintf(buf, sizeof(buf), "output check: block %u is stored with a compression the engine does not decode", hV.error_where);
    return Fail(YBGPU_NOT_SUPPORTED, buf);
  }
  if (hV.error) fail = std::min(fail, verify_pack(hV.error_where, 0, VERIFY_COMPRESSED));
  if (fail == ~0ull && job && hV.n_counted != I.n_out) fail = verify_pack(nb, 0, VERIFY_COUNT);
  if (fail == ~0ull) return YBGPU_OK;
  result->failure_kind = static_cast<uint32_t>(fail & 15);
  result->failure_block = static_cast<uint32_t>(fail >> 32);
  result->failure_entry = static_cast<uint32_t>((fail >> 4) & 0x0fffffffu);
  char buf[256];
  snprintf(buf, sizeof(buf), "output check failed: %s at data block %u, entry %u (%llu blocks, %llu entries parsed)", VerifyKindName(result->failure_kind),
           result->failure_block, result->failure_entry, static_cast<unsigned long long>(nb), static_cast<unsigned long long>(hV.n_counted));
  return Fail(result->failure_kind == VERIFY_KEY_TOO_LONG ? YBGPU_NOT_SUPPORTED : YBGPU_CORRUPTION, buf);
}

ybgpu_status Engine::VerifyOutput(ybgpu_output_check* result) {
  if (!ran_) return Fail(YBGPU_ILLEGAL_STATE, "job has not run");
  Impl& I = *impl_;
  CUDA_TRY(cudaSetDevice(opt_.device));
  ybgpu_status s = VerifyTable(I.out_file, I.out_file_len, I.d_block_off, nullptr, I.n_blocks, opt_.output_key_encoding, true, result);
  if (s == YBGPU_OK) stats_.path_flags |= YBGPU_PATH_OUTPUT_VERIFIED;
  return s;
}

ybgpu_status Engine::VerifySst(const uint8_t* data, uint64_t len, const ybgpu_block_handle* handles, uint64_t nh, int key_encoding,
                               ybgpu_output_check* result) {
  Impl& I = *impl_;
  memset(result, 0, sizeof(*result));
  if (key_encoding != YBGPU_KEY_ENCODING_SHARED_PREFIX && key_encoding != YBGPU_KEY_ENCODING_THREE_SHARED_PARTS)
    return Fail(YBGPU_NOT_SUPPORTED, "data block key-value encoding format " + std::to_string(key_encoding) + " is not decoded by the engine");
  if (nh >= (1ull << 32)) return Fail(YBGPU_NOT_SUPPORTED, "too many data blocks in one file");
  std::vector<unsigned long long> off(nh); std::vector<uint32_t> sz(nh);
  for (uint64_t i = 0; i < nh; i++) {
    if (handles[i].offset > len || handles[i].size > len - handles[i].offset || len - handles[i].offset - handles[i].size < 5)
      return Fail(YBGPU_CORRUPTION, "block handle outside the data file");
    if (handles[i].size >= (1ull << 31)) return Fail(YBGPU_NOT_SUPPORTED, "data block too large");
    off[i] = handles[i].offset; sz[i] = static_cast<uint32_t>(handles[i].size);
  }
  if (nh == 0) return YBGPU_OK;
  CUDA_TRY(cudaSetDevice(opt_.device));
  VerifyScratch T(I.mem, I.stream);
  uint8_t* d = nullptr; unsigned long long* d_off = nullptr; uint32_t* d_sz = nullptr;
  CUDA_TRY(T.Alloc(&d, len + 64)); CUDA_TRY(T.Alloc(&d_off, nh)); CUDA_TRY(T.Alloc(&d_sz, nh));
  CUDA_TRY(cudaMemsetAsync(d, 0, 16, I.stream));
  CUDA_TRY(ChunkedCopyAsync(d + 16, data, len, cudaMemcpyHostToDevice, I.stream));
  CUDA_TRY(cudaMemsetAsync(d + 16 + len, 0, 48, I.stream));
  CUDA_TRY(cudaMemcpyAsync(d_off, off.data(), nh * 8, cudaMemcpyHostToDevice, I.stream));
  CUDA_TRY(cudaMemcpyAsync(d_sz, sz.data(), nh * 4, cudaMemcpyHostToDevice, I.stream));
  const ybgpu_status s = VerifyTable(d + 16, len, d_off, d_sz, static_cast<uint32_t>(nh), key_encoding, false, result);
  CUDA_TRY(cudaStreamSynchronize(I.stream));               // the host arrays and the caller's file are free again
  return s;
}

}  // namespace ybgpu

extern "C" int32_t ybgpu_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}
