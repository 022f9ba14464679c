// verify_kernels.cuh — V: the output check (DBOptions::paranoid_file_checks, compaction_job.cc:932-971) on the GPU.
//
// The block assembler derives every trailer from checksums of the input values and reads no block back, so nothing in a
// job looks at the bytes it stored. These kernels do, working from what a reader of the file has — the data image in
// HBM and the block offsets / sizes — in the order ReadBlock + BlockIter would:
//   k_verify_sizes     block sizes from the offsets, trailer type bytes counted (compressed blocks)
//   k_crc_blocks       (encode_kernels.cuh, mode 2) masked CRC32C of the stored bytes + type against the trailer
//   k_snappy_sizes / k_snappy_decode (snappy_kernels.cuh, lz4_kernels.cuh) compressed blocks into a scratch image
//   k_verify_blocks    one warp per block, one lane per restart interval (the walker scheme of k_prepass): every entry
//                      parsed and its key rebuilt by verify_interval (dev_logic.cuh, shared with the CPU tests), keys
//                      strictly ascending inside the interval, across intervals, and into the next block; for a job,
//                      entry i of the table against survivor i (key, value length, value bytes from where the merge
//                      left them), the block's entry count against the block cuts and the first / last key of the file
//                      against the boundary records the index is written from.
// One failure word per table: atomicMin of verify_pack(block, entry, kind), so the report does not depend on scheduling.
//
// Included by engine.cu only.
#pragma once

namespace ybgpu {

struct VerifyView {
  const uint8_t* data;               // the table as a reader sees it after uncompression (the stored table if no block is compressed)
  const unsigned long long* off;     // [nblocks] block offsets in `data`
  const uint32_t* size;              // [nblocks] contents sizes (without the trailer)
  uint32_t nblocks;
  int key_encoding;
  uint32_t ri;                       // restart interval the table was written with (every interval but a block's last is full); 0 = unknown
  uint8_t* keybuf;                   // two key buffers of kstride bytes per thread of the grid
  uint32_t kstride, kcap;            // kcap: longest key rebuilt
  // the merge result (jobs; null / unused for a table that came from outside)
  const uint32_t* block_first;       // [nblocks] first output entry of every block
  const uint8_t* boundary;           // k_boundary_keys records, stride boundary_stride: slot 2b = last key of block b, slot 2 nblocks = first key of the file
  uint32_t boundary_stride;
};

// Entry `i` of the table against survivor `i`: what k_encode_* were asked to write, read from the merge's own state.
struct VerifySurvivors {
  const EncView* E; int S;
  __device__ bool operator()(uint32_t j, const uint8_t* key, uint32_t klen, const uint8_t* val, uint32_t vlen) const {
    if (j >= E->n) return false;
    const Desc d = E->kept[j];
    if (d.klen != klen || d.vlen_out != vlen) return false;
    const RunView& run = E->runs[d.run];
    const uint32_t idx = d.gid - run.gid_base;
    const uint8_t* rec = run.rec + static_cast<size_t>(idx) * S;
    const uint32_t ulen = klen - 8u;
    for (uint32_t i = 0; i < ulen; i++) if (key[i] != rec[i]) return false;
    const uint64_t suffix = kept_suffix(rec, d, S);
    for (int i = 0; i < 8; i++) if (key[ulen + i] != static_cast<uint8_t>(suffix >> (8 * i))) return false;
    if (d.flags & ENT_VAL_TOMBSTONE) return vlen == 1 && val[0] == 'X';
    const uint8_t* vs = run.data + run.val_off[idx];
    uint32_t i = 0;
    if (d.flags & ENT_VAL_REENCODE) {
      const ValueRewrite& rw = E->rewrites[d.rewrite_slot];
      if (rw.prefix_len > vlen) return false;
      for (; i < rw.prefix_len; i++) if (val[i] != rw.prefix[i]) return false;
      vs += rw.skip; val += i; vlen -= i; i = 0;
    }
    if (((reinterpret_cast<uintptr_t>(vs) ^ reinterpret_cast<uintptr_t>(val)) & 3) == 0) {   // same phase: whole words
      for (; i < vlen && (reinterpret_cast<uintptr_t>(val + i) & 3); i++) if (val[i] != vs[i]) return false;
      for (; i + 4 <= vlen; i += 4)
        if (*reinterpret_cast<const uint32_t*>(val + i) != *reinterpret_cast<const uint32_t*>(vs + i)) return false;
    }
    for (; i < vlen; i++) if (val[i] != vs[i]) return false;
    return true;
  }
};

// Contents sizes of the blocks of a table stored back to back (a job's output), and how many are stored compressed.
__global__ void __launch_bounds__(256) k_verify_sizes(const uint8_t* file, const unsigned long long* off /*[n+1]*/, const uint32_t* size_in, uint32_t nblocks,
                                                      uint32_t* size_out, JobDev* J) {
  uint32_t comp = 0;
  for (uint32_t b = blockIdx.x * blockDim.x + threadIdx.x; b < nblocks; b += gridDim.x * blockDim.x) {
    const uint32_t size = size_in ? size_in[b] : static_cast<uint32_t>(off[b + 1] - off[b] - 5);
    if (size_out) size_out[b] = size;
    comp += file[off[b] + size] != 0;
  }
  comp = __reduce_add_sync(0xffffffffu, comp);
  if ((threadIdx.x & 31) == 0 && comp) atomicAdd(&J->n_compressed, comp);
}

constexpr int VERIFY_THREADS = 128;

template <bool JOB>
__global__ void __launch_bounds__(VERIFY_THREADS) k_verify_blocks(VerifyView V, EncView E, int S, JobDev* J) {
  const int lane = threadIdx.x & 31;
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t warp = tid >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  uint8_t* buf0 = V.keybuf + static_cast<size_t>(tid) * 2 * V.kstride;
  uint8_t* buf1 = buf0 + V.kstride;
  unsigned long long entries = 0;
  for (uint32_t b = warp; b < V.nblocks; b += nwarps) {
    const uint8_t* blk = V.data + V.off[b];
    const uint32_t size = V.size[b];
    unsigned long long fail = ~0ull;                       // this lane's lowest failure in the block
    uint32_t count = 0;
    uint32_t nres = 0, roff = 0;
    if (!verify_block_layout(blk, size, &nres, &roff)) {
      fail = verify_pack(b, 0, VERIFY_PARSE);
    } else {
      const uint32_t first_entry = JOB ? V.block_first[b] : 0u;
      unsigned long long carry_key = 0; uint32_t carry_klen = 0;   // last key of the previous round's last interval (0 = none)
      VerifyWalk w{};
      for (uint32_t r0 = 0; r0 < nres; r0 += 32) {
        const uint32_t r = r0 + lane;
        const bool active = r < nres;
        uint32_t p = 0, end = 0;
        const bool bounds_ok = active && verify_interval_bounds(blk, nres, roff, r, &p, &end);
        const uint8_t* fkey = nullptr; uint32_t fklen = 0;
        const bool have_first = bounds_ok && verify_restart_key(blk, p, end, V.key_encoding, &fkey, &fklen);
        // lane 0 meets the previous round's last key before lane 31 reuses its buffers
        bool join_bad = lane == 0 && have_first && carry_klen &&
                        cmp_internal_keys(reinterpret_cast<const uint8_t*>(carry_key), carry_klen, fkey, fklen) >= 0;
        __syncwarp();
        w.n = 0; w.kind = VERIFY_OK; w.last_key = nullptr; w.last_klen = 0;
        if (bounds_ok) {
          if (JOB) verify_interval(blk, p, end, V.key_encoding, buf0, buf1, V.kcap, first_entry + r * V.ri, VerifySurvivors{&E, S}, &w);
          else verify_interval(blk, p, end, V.key_encoding, buf0, buf1, V.kcap, 0u, VerifyNoExpect{}, &w);
        } else if (active) {
          w.kind = VERIFY_PARSE;
        }
        __syncwarp();                                      // the lanes' key buffers are visible to their neighbours
        uint32_t incl = w.n;
        for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += y; }
        const uint32_t base = count + incl - w.n;
        if (w.kind != VERIFY_OK) fail = min(fail, verify_pack(b, base + w.n, w.kind));
        else if (V.ri && (r + 1 < nres ? w.n != V.ri : w.n > V.ri)) fail = min(fail, verify_pack(b, base, VERIFY_COUNT));
        // the interval's first key against the last key of the interval before it
        const bool whole = w.kind == VERIFY_OK && w.n > 0;
        const unsigned long long nb_key = __shfl_up_sync(0xffffffffu, reinterpret_cast<unsigned long long>(w.last_key), 1);
        const uint32_t nb_klen = __shfl_up_sync(0xffffffffu, whole ? w.last_klen : 0u, 1);
        if (lane > 0 && have_first && nb_klen && cmp_internal_keys(reinterpret_cast<const uint8_t*>(nb_key), nb_klen, fkey, fklen) >= 0) join_bad = true;
        if (join_bad) fail = min(fail, verify_pack(b, base, VERIFY_ORDER));
        count += __shfl_sync(0xffffffffu, incl, 31);
        carry_key = __shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(w.last_key), 31);
        carry_klen = __shfl_sync(0xffffffffu, whole ? w.last_klen : 0u, 31);
      }
      // the lane that walked the last interval holds the block's last key
      const bool last_lane = lane == static_cast<int>((nres - 1) & 31) && w.kind == VERIFY_OK && w.n > 0;
      if (last_lane && b + 1 < V.nblocks) {
        const uint8_t* nblk = V.data + V.off[b + 1];
        uint32_t nn = 0, nroff = 0, np = 0, nend = 0;
        const uint8_t* nkey = nullptr; uint32_t nklen = 0;
        if (verify_block_layout(nblk, V.size[b + 1], &nn, &nroff) && verify_interval_bounds(nblk, nn, nroff, 0, &np, &nend) &&
            verify_restart_key(nblk, np, nend, V.key_encoding, &nkey, &nklen) && cmp_internal_keys(w.last_key, w.last_klen, nkey, nklen) >= 0)
          fail = min(fail, verify_pack(b + 1, 0, VERIFY_ORDER));
      }
      if (JOB) {
        // a walk that stopped early has its own report; the count is judged on blocks that parsed to their end
        const uint32_t expect = (b + 1 < V.nblocks ? V.block_first[b + 1] : E.n) - first_entry;
        if (!__any_sync(0xffffffffu, fail != ~0ull) && count != expect) fail = min(fail, verify_pack(b, min(count, expect), VERIFY_COUNT));
        // FileMetaData::smallest / largest and the index are written from these records
        if (b == 0 && lane == 0) {
          const uint8_t* rec = V.boundary + static_cast<size_t>(V.nblocks) * 2 * V.boundary_stride;
          uint32_t p0 = 0, e0 = 0; const uint8_t* k0 = nullptr; uint32_t kl0 = 0;
          if (verify_interval_bounds(blk, nres, roff, 0, &p0, &e0) && verify_restart_key(blk, p0, e0, V.key_encoding, &k0, &kl0) &&
              (ld_u16(rec) != kl0 || cmp_raw(rec + 2, kl0, k0, kl0) != 0))
            fail = min(fail, verify_pack(0, 0, VERIFY_CONTENTS));
        }
        if (last_lane) {
          const uint8_t* rec = V.boundary + static_cast<size_t>(b) * 2 * V.boundary_stride;
          if (ld_u16(rec) != w.last_klen || cmp_raw(rec + 2, w.last_klen, w.last_key, w.last_klen) != 0)
            fail = min(fail, verify_pack(b, count ? count - 1 : 0, VERIFY_CONTENTS));
        }
      }
      __syncwarp();                                        // the next block's walk reuses the key buffers
    }
    for (int o = 16; o; o >>= 1) fail = min(fail, __shfl_xor_sync(0xffffffffu, fail, o));
    if (lane == 0 && fail != ~0ull) atomicMin(&J->verify_fail, fail);
    entries += count;
  }
  if (lane == 0 && entries) atomicAdd(&J->n_counted, entries);
}

}  // namespace ybgpu
