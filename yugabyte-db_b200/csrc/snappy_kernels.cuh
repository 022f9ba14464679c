// snappy_kernels.cuh — Snappy-compressed input data blocks (SURVEY.md 8f-2).
//
// DocDB's production default is kSnappyCompression (docdb_rocksdb_util.cc:184): a data block is stored compressed
// when that saves at least 12.5 % (block_based_table_builder.cc:109-131), its trailer's type byte says so, and
// ReadBlock uncompresses it after the checksum check (table/format.cc:441-500 UncompressBlockContents). Here the
// compressed blocks of all inputs are uncompressed once, on the GPU, into a second image of the input files (blocks
// that were stored raw are copied); every later kernel runs on that image unchanged.
//
// Format (snappy's format_description.txt; the library itself lives in yugabyte-db-thirdparty and is not vendored):
// varint32 uncompressed length, then elements — tag & 3 == 0: literal (length - 1 in the tag's upper six bits, or in
// the 1..4 following bytes for 60..63), 1: copy with 11-bit offset and length 4..11, 2 / 3: copy with 16- / 32-bit
// offset and length 1..64. A copy may overlap its own output (run-length patterns).
//
// One warp per block. Every lane parses the element stream redundantly (all lanes read the same tag bytes: one
// broadcast load), so the control flow is uniform and nothing is shuffled; the bytes of a literal or a copy are
// spread over the lanes. A copy whose offset is at least 32 proceeds in rounds of 32 bytes (a round only reads what
// earlier rounds or elements wrote), a closer one is a repeating pattern of bytes that were written before the
// element began. __syncwarp() orders the lanes' global stores and loads between rounds.
//
// k_snappy_sizes and k_snappy_decode take every codec the engine reads in the same pass: raw blocks are copied, LZ4 /
// LZ4HC blocks (trailer type 4 / 5, the same varint32 preamble) are decoded by lz4_kernels.cuh lz4_warp_decode, so a
// job over tables written with different codecs still builds one uncompressed image.
//
// Included by engine.cu (and, for the CPU tests, by tests/host_harness); it includes lz4_kernels.cuh at its end.
#pragma once

namespace ybgpu {

struct SnapView {
  const RunView* runs;
  const uint32_t* blk_base;          // [k+1]
  unsigned long long* out_off;       // [total blocks + 1] sizes (contents + 5-byte trailer) -> exclusive prefix -> offsets
  uint32_t* usize;                   // [total blocks] uncompressed contents size
  uint8_t* out;                      // the uncompressed image (k_snappy_decode)
  int k;
};

__device__ __forceinline__ int snap_varint32(const uint8_t* p, uint32_t avail, uint32_t* v) {
  uint32_t r = 0;
  for (int i = 0; i < 5 && static_cast<uint32_t>(i) < avail; i++) {
    const uint32_t b = p[i];
    r |= (b & 127) << (7 * i);
    if (!(b & 128)) { *v = r; return i + 1; }
  }
  return 0;
}

// Per block: the size of its uncompressed contents.
__global__ void __launch_bounds__(256) k_snappy_sizes(SnapView V, JobDev* J) {
  const uint32_t total = V.blk_base[V.k];
  for (uint32_t gb = blockIdx.x * blockDim.x + threadIdx.x; gb < total; gb += gridDim.x * blockDim.x) {
    int r = 0;
    while (V.blk_base[r + 1] <= gb) r++;
    const RunView& run = V.runs[r];
    const uint32_t b = gb - V.blk_base[r];
    const uint8_t* blk = run.data + run.blk_off[b];
    const uint32_t size = run.blk_size[b];
    const uint8_t type = blk[size];
    uint32_t u = size;
    if (type == 1 || type == 4 || type == 5) {            // Snappy, LZ4, LZ4HC: the same varint32 preamble
      if (!snap_varint32(blk, size, &u) || u >= (1u << 30)) { dev_fail(J, DEV_ERR_BAD_BLOCK, b); u = 0; }
    } else if (type != 0) {
      dev_fail(J, DEV_ERR_COMPRESSED, b);
    }
    V.usize[gb] = u;
    V.out_off[gb] = static_cast<unsigned long long>(u) + 5;
  }
}

// lz4_kernels.cuh: one LZ4 block by one warp (the preamble already read); false on a malformed stream
__device__ __forceinline__ bool lz4_warp_decode(const uint8_t* src, uint32_t size, uint32_t ip, uint8_t* dst, uint32_t ulen, int lane);

// Every block of every input, whatever its codec: raw blocks are copied, Snappy and LZ4 (LZ4HC) blocks decoded.
__global__ void __launch_bounds__(128) k_snappy_decode(SnapView V, JobDev* J) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t total = V.blk_base[V.k];
  for (uint32_t gb = warp; gb < total; gb += nwarps) {
    int r = 0;
    while (V.blk_base[r + 1] <= gb) r++;
    const RunView& run = V.runs[r];
    const uint32_t b = gb - V.blk_base[r];
    const uint8_t* src = run.data + run.blk_off[b];
    const uint32_t size = run.blk_size[b];
    const uint32_t ulen = V.usize[gb];
    uint8_t* dst = V.out + V.out_off[gb];
    const uint8_t type = src[size];
    if (type == 0) {
      for (uint32_t i = lane; i < size; i += 32) dst[i] = src[i];
    } else if (type == 1) {
      uint32_t u;
      uint32_t ip = static_cast<uint32_t>(snap_varint32(src, size, &u));
      uint32_t op = 0;
      bool bad = ip == 0;
      while (!bad && ip < size) {
        const uint32_t tag = src[ip++];
        const uint32_t kind = tag & 3;
        if (kind == 0) {
          uint32_t len = tag >> 2;
          if (len >= 60) {
            const uint32_t nb = len - 59;
            if (size - ip < nb) { bad = true; break; }
            len = 0;
            for (uint32_t i = 0; i < nb; i++) len |= static_cast<uint32_t>(src[ip + i]) << (8 * i);
            ip += nb;
          }
          len += 1;
          if (size - ip < len || ulen - op < len) { bad = true; break; }
          for (uint32_t i = lane; i < len; i += 32) dst[op + i] = src[ip + i];
          ip += len; op += len;
        } else {
          uint32_t len, off;
          if (kind == 1) { if (ip >= size) { bad = true; break; } len = 4 + ((tag >> 2) & 7); off = ((tag >> 5) << 8) | src[ip]; ip += 1; }
          else if (kind == 2) { if (size - ip < 2) { bad = true; break; } len = 1 + (tag >> 2); off = src[ip] | (static_cast<uint32_t>(src[ip + 1]) << 8); ip += 2; }
          else {
            if (size - ip < 4) { bad = true; break; }
            len = 1 + (tag >> 2);
            off = src[ip] | (static_cast<uint32_t>(src[ip + 1]) << 8) | (static_cast<uint32_t>(src[ip + 2]) << 16) | (static_cast<uint32_t>(src[ip + 3]) << 24);
            ip += 4;
          }
          if (off == 0 || off > op || ulen - op < len) { bad = true; break; }
          __syncwarp();                                        // what earlier elements wrote is visible to every lane
          if (off >= 32) {
            for (uint32_t base = 0; base < len; base += 32) {
              const uint32_t i = base + lane;
              if (i < len) dst[op + i] = dst[op - off + i];
              __syncwarp();
            }
          } else {
            for (uint32_t i = lane; i < len; i += 32) dst[op + i] = dst[op - off + (i % off)];
          }
          op += len;
        }
      }
      __syncwarp();
      if (bad || op != ulen) { if (lane == 0) dev_fail(J, DEV_ERR_BAD_BLOCK, b); }
    } else if (type == 4 || type == 5) {
      uint32_t u;
      const uint32_t ip = static_cast<uint32_t>(snap_varint32(src, size, &u));
      const bool ok = ip != 0 && lz4_warp_decode(src, size, ip, dst, ulen, lane);
      __syncwarp();
      if (!ok && lane == 0) dev_fail(J, DEV_ERR_BAD_BLOCK, b);
    }
    // the image's trailer: stored raw; the checksum of the stored (compressed) bytes was verified before
    if (lane < 5) dst[ulen + lane] = 0;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Snappy-compressed OUTPUT data blocks (SURVEY.md 8a-17: BlockBasedTableBuilder::WriteBlock -> CompressBlock,
// block_based_table_builder.cc:115-131,630-655). The block assembler writes the table uncompressed (contents +
// trailer, back to back); k_snappy_compress then encodes every block into a scratch image at the same offsets and
// decides per block whether the compressed form is kept (GoodCompressionRatio, :109-112: shorter than 7/8 of the
// contents — an encoding that reaches that bound is abandoned on the spot, so the scratch never overflows a block's
// slot); the kept sizes are prefix-summed into the final block offsets and k_snappy_gather moves each block's stored
// form (compressed + type 1 + checksum of the compressed bytes, or the raw block with the trailer it already has).
//
// Encoder (one warp per block; identical element for element to host_sst.cc SnappyCompress, which writes the index
// blocks of the same table): 64 KB fragments; a table of 2^12 fragment-relative positions per warp in shared memory,
// keyed by a multiplicative hash of the four bytes at a position. The scalar algorithm visits positions one by one:
// the slot's previous occupant is the match candidate, the position takes the slot. Here 32 consecutive positions are
// tried at once: a lane's candidate is the nearest lower lane with the same hash (__match_any_sync) or else the
// slot's occupant; the lowest lane that finds a four-byte match wins, lanes up to and including it take their slots
// (the highest lane of every hash group), the lanes behind it are covered by the match and do not count as visited —
// exactly the scalar order of events. The match is extended 32 bytes per step; literal bytes are moved with
// word-wide copies.
constexpr int SNAPC_WARPS = 4;
constexpr uint32_t SNAPC_HASH_BITS = 12;
constexpr uint32_t SNAPC_FRAGMENT = 65536;

struct SnapCompView {
  const uint8_t* raw;                  // assembled table: block b at raw_off[b], contents + 5-byte trailer
  const unsigned long long* raw_off;   // [nblocks + 1]
  uint8_t* comp;                       // scratch image, same offsets
  uint32_t* csize;                     // [nblocks] compressed contents size; 0 = the block stays raw
  unsigned long long* fsize;           // [nblocks + 1] stored size incl. trailer -> exclusive prefix sum -> final offsets
  uint8_t* out;                        // final table (k_snappy_gather)
  uint32_t nblocks;
};

__device__ __forceinline__ uint32_t snapc_literal_header(uint32_t len, uint32_t* nbytes) {
  const uint32_t l1 = len - 1;
  if (l1 < 60) { *nbytes = 1; return l1 << 2; }
  if (l1 < 256) { *nbytes = 2; return (60u << 2) | (l1 << 8); }
  *nbytes = 3; return (61u << 2) | (l1 << 8);            // l1 <= 65535: a literal never crosses a fragment
}

// Four bytes at any address: the two aligned words around them (reads at most 7 bytes past p, inside the block's
// trailer or the buffer's padding).
__device__ __forceinline__ uint32_t snapc_load32(const uint8_t* p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint32_t* q = reinterpret_cast<const uint32_t*>(a & ~static_cast<uintptr_t>(3));
  return __funnelshift_r(__ldg(q), __ldg(q + 1), static_cast<uint32_t>(a & 3) * 8);   // the assembled table is read-only here
}

// What a lane knows about its position of a batch before the table is consulted.
struct SnapcBatch {
  uint32_t w, h, tag, grp;
  bool act;
};

// VARIANT 0: hash groups by __match_any_sync. 1: by one ballot per hash bit (twelve independent votes). 2: as 1, and the
// NEXT batch (its bytes, hashes and groups, none of which depend on the table) is prepared before the current one is
// resolved, so that the loads and votes of one batch overlap the table round trip of the other; a match discards it.
template <int VARIANT>
__device__ __forceinline__ SnapcBatch snapc_prepare(const uint8_t* f, uint32_t i, uint32_t m, int lane) {
  const uint32_t FULL = 0xffffffffu;
  SnapcBatch B;
  const uint32_t pos = i + lane;
  B.act = pos + 4 <= m && pos >= i;
  B.w = 0; B.h = 0x10000u + lane; B.tag = 0;            // idle lanes: a hash group of their own
  if (B.act) {
    B.w = snapc_load32(f + pos);
    const uint32_t prod = B.w * 0x1e35a7bdu;
    B.h = prod >> (32 - SNAPC_HASH_BITS); B.tag = (prod >> (24 - SNAPC_HASH_BITS)) & 0xffu;
  }
  if (VARIANT == 0) {
    B.grp = __match_any_sync(FULL, B.h);
  } else {
#if defined(__CUDA_ARCH__)                                // (the kernel source is also compiled for the CPU by tests/host_harness/warp_emu.cc)
    if (lane == 0 && i + 288 < m) asm volatile("prefetch.global.L2 [%0];" :: "l"(f + i + 256));
#endif
    uint32_t g = __ballot_sync(FULL, B.act);
#pragma unroll
    for (uint32_t bit = 0; bit < SNAPC_HASH_BITS; bit++) {
      const bool one = (B.h >> bit) & 1u;
      const uint32_t v = __ballot_sync(FULL, one);
      g &= one ? v : ~v;
    }
    B.grp = B.act ? g : (1u << lane);
  }
  return B;
}

// Per warp: the slot's position and eight more bits of the occupant's hash product. A candidate whose tag differs
// cannot hold the same four bytes, so its bytes (a scattered read of the block: 32 lanes, 32 sectors) are fetched
// only when the tag agrees — with nothing to find that is one batch in eight instead of every batch. Zeroed at every
// fragment's start.
__device__ __forceinline__ void snapc_clear_table(uint16_t* T, uint8_t* G, int lane) {
  __syncwarp();
  for (uint32_t i = lane; i < (1u << SNAPC_HASH_BITS) / 2; i += 32) reinterpret_cast<uint32_t*>(T)[i] = 0;
  for (uint32_t i = lane; i < (1u << SNAPC_HASH_BITS) / 4; i += 32) reinterpret_cast<uint32_t*>(G)[i] = 0;
  __syncwarp();
}

// The search of both output encoders (k_snappy_compress, and k_lz4_compress in lz4_kernels.cuh). From position i of the
// fragment f on, batches of 32 positions p with p + 4 <= smax are resolved against the table until one finds a match.
// Returns false when no position is left; else the match (*mpos, its candidate *cand, *len: extended while
// mpos + len < emax), with i moved behind it and cur holding the batch there. Snappy passes the fragment's end for both
// limits, LZ4 its end-of-block limits (positions up to n - 12, matches ending by n - 5).
template <int VARIANT>
__device__ __forceinline__ bool snapc_next_match(const uint8_t* f, uint32_t& i, SnapcBatch& cur, uint32_t smax, uint32_t emax, uint16_t* T,
                                                 uint8_t* G, int lane, uint32_t* mpos_out, uint32_t* cand_out, uint32_t* len_out) {
  const uint32_t FULL = 0xffffffffu;
  while (i + 4 <= smax) {
    SnapcBatch nxt;
    if (VARIANT == 2) nxt = snapc_prepare<VARIANT>(f, i + 32, smax, lane);
    const uint32_t pos = i + lane;
    const bool act = cur.act;
    const uint32_t w = cur.w, h = cur.h, tag = cur.tag, grp = cur.grp;
    const uint32_t lower = grp & ((1u << lane) - 1u);
    const int nearest = lower ? 31 - __clz(lower) : lane;                          // the nearest lower lane of the group
    const uint32_t w_nearest = __shfl_sync(FULL, w, nearest);
    uint32_t cand = 0;
    bool hit = false;
    if (act) {
      if (lower) { cand = i + nearest; hit = w_nearest == w; }
      else { cand = T[h]; hit = cand < pos && G[h] == tag && snapc_load32(f + cand) == w; }
    }
    const uint32_t hits = __ballot_sync(FULL, hit);
    const uint32_t upto = hits ? static_cast<uint32_t>(__ffs(hits) - 1) : 31u;     // lanes <= upto are visited
    __syncwarp();
    if (act && static_cast<uint32_t>(lane) <= upto) {
      const uint32_t g = grp & (0xffffffffu >> (31 - upto));
      if (31 - __clz(g) == lane) { T[h] = static_cast<uint16_t>(pos); G[h] = static_cast<uint8_t>(tag); }
    }
    __syncwarp();
    if (!hits) {
      i += 32;
      if (VARIANT == 2) cur = nxt; else cur = snapc_prepare<VARIANT>(f, i, smax, lane);
      continue;
    }
    const uint32_t mpos = i + upto;
    const uint32_t c = __shfl_sync(FULL, cand, upto);
    uint32_t len = 4;
    for (;;) {                                            // extend: 32 bytes per step
      const uint32_t q = mpos + len + lane;
      const bool same = q < emax && f[c + len + lane] == f[q];
      const uint32_t differ = __ballot_sync(FULL, !same);
      if (differ) { len += __ffs(differ) - 1; break; }
      len += 32;
    }
    *mpos_out = mpos; *cand_out = c; *len_out = len;
    i = mpos + len;
    cur = snapc_prepare<VARIANT>(f, i, smax, lane);
    return true;
  }
  return false;
}

template <int VARIANT>
__global__ void __launch_bounds__(SNAPC_WARPS * 32) k_snappy_compress(SnapCompView V) {
  __shared__ uint16_t s_pos[SNAPC_WARPS][1u << SNAPC_HASH_BITS];   // the hash table (snapc_clear_table)
  __shared__ uint8_t s_tag[SNAPC_WARPS][1u << SNAPC_HASH_BITS];
  const int lane = threadIdx.x & 31;
  uint16_t* T = s_pos[threadIdx.x >> 5];
  uint8_t* G = s_tag[threadIdx.x >> 5];
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t b = warp; b < V.nblocks; b += nwarps) {
    const unsigned long long o = V.raw_off[b];
    const unsigned long long n64 = V.raw_off[b + 1] - o - 5;
    const uint8_t* in = V.raw + o;
    uint8_t* out = V.comp + o;
    const uint32_t n = static_cast<uint32_t>(n64);
    const uint32_t limit = n - n / 8u;                    // kept only if the stream is SHORTER than this
    bool give_up = n64 >= 0x7fffffffull;                  // kCompressionSizeLimit (:642)
    uint32_t op = 0;
    if (!give_up) {                                       // varint32 preamble: the uncompressed length
      uint32_t v = n;
      while (v >= 128) { if (lane == 0) out[op] = static_cast<uint8_t>(v | 128); v >>= 7; op++; }
      if (lane == 0) out[op] = static_cast<uint8_t>(v);
      op++;
      if (op >= limit) give_up = true;
    }
    for (uint32_t fs = 0; fs < n && !give_up; fs += SNAPC_FRAGMENT) {
      const uint8_t* f = in + fs;
      const uint32_t m = min(n - fs, SNAPC_FRAGMENT);
      snapc_clear_table(T, G, lane);
      uint32_t lit = 0, i = 0, mpos, c, len;
      SnapcBatch cur = snapc_prepare<VARIANT>(f, 0, m, lane);
      while (snapc_next_match<VARIANT>(f, i, cur, m, m, T, G, lane, &mpos, &c, &len)) {
        // ---- the literal in front of the match
        if (mpos > lit) {
          const uint32_t L = mpos - lit;
          uint32_t hb; const uint32_t hdr = snapc_literal_header(L, &hb);
          if (op + hb + L >= limit) { give_up = true; break; }
          if (lane < static_cast<int>(hb)) out[op + lane] = static_cast<uint8_t>(hdr >> (8 * lane));
          warp_copy(out + op + hb, f + lit, L, lane);
          op += hb + L;
        }
        // ---- the copy: pieces of 64 bytes while at least 4 remain behind them, then one or two closing pieces
        const uint32_t off = mpos - c;
        const uint32_t nfull = len >= 68 ? (len - 68) / 64 + 1 : 0;
        uint32_t left = len - 64 * nfull;                 // 4..67
        unsigned long long closing = 0; uint32_t cb = 0;  // the closing pieces' bytes, packed
        while (left) {
          uint32_t l = min(left, 64u);
          if (left > l && left - l < 4) l = left - 4;
          if (l <= 11 && off < 2048) {
            closing |= static_cast<unsigned long long>(1u | ((l - 4) << 2) | ((off >> 8) << 5) | ((off & 0xff) << 8)) << (8 * cb);
            cb += 2;
          } else {
            closing |= static_cast<unsigned long long>(2u | ((l - 1) << 2) | (off << 8)) << (8 * cb);
            cb += 3;
          }
          left -= l;
        }
        if (op + 3 * nfull + cb >= limit) { give_up = true; break; }
        for (uint32_t j = lane; j < nfull; j += 32) {
          uint8_t* e = out + op + 3 * j;
          e[0] = static_cast<uint8_t>(2u | (63u << 2)); e[1] = static_cast<uint8_t>(off); e[2] = static_cast<uint8_t>(off >> 8);
        }
        op += 3 * nfull;
        if (lane < static_cast<int>(cb)) out[op + lane] = static_cast<uint8_t>(closing >> (8 * lane));
        op += cb;
        lit = mpos + len;
      }
      if (!give_up && m > lit) {                          // the fragment's closing literal
        const uint32_t L = m - lit;
        uint32_t hb; const uint32_t hdr = snapc_literal_header(L, &hb);
        if (op + hb + L >= limit) { give_up = true; break; }
        if (lane < static_cast<int>(hb)) out[op + lane] = static_cast<uint8_t>(hdr >> (8 * lane));
        warp_copy(out + op + hb, f + lit, L, lane);
        op += hb + L;
      }
    }
    const bool keep = !give_up && op < limit;
    if (lane == 0) {
      if (keep) out[op] = 1;                              // the trailer's type byte: kSnappyCompression
      V.csize[b] = keep ? op : 0u;
      V.fsize[b] = (keep ? static_cast<unsigned long long>(op) : n64) + 5ull;
    }
  }
}

// Moves every block's stored form to its final place; compressed blocks get their checksum here (over the
// compressed bytes and the type byte, masked: WriteRawBlock, block_based_table_builder.cc:684-689). Codec-agnostic:
// the encoder (k_snappy_compress or lz4_kernels.cuh k_lz4_compress) has written the type byte behind the stream.
__global__ void __launch_bounds__(256) k_snappy_gather(SnapCompView V) {
  __shared__ uint32_t tab0[256];
  __shared__ uint32_t s32[4][256];
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) (&s32[0][0])[i] = (&g_crc_s32[0][0])[i];
  tab0[threadIdx.x] = g_crc_tab[0][threadIdx.x];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const uint32_t kc = g_crc_xpow8[4 * (lane + 1)];
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t b = warp; b < V.nblocks; b += nwarps) {
    const unsigned long long o = V.raw_off[b];
    const uint32_t cs = V.csize[b];
    uint8_t* dst = V.out + V.fsize[b];
    if (!cs) {
      const unsigned long long len = V.raw_off[b + 1] - o;      // contents + trailer
      const uint8_t* src = V.raw + o;
      for (unsigned long long done = 0; done < len; done += 1u << 30) {
        const uint32_t part = static_cast<uint32_t>(len - done < (1ull << 30) ? len - done : (1ull << 30));
        warp_copy(dst + done, src + done, part, lane);
      }
    } else {
      const uint8_t* src = V.comp + o;
      warp_copy(dst, src, cs + 1, lane);
      const uint32_t crc = crc_mask(warp_crc32c_strided(src, static_cast<uint64_t>(cs) + 1, lane, tab0, s32, kc));
      if (lane < 4) dst[cs + 1 + lane] = static_cast<uint8_t>(crc >> (8 * lane));
    }
  }
}

}  // namespace ybgpu

// The LZ4 kernels come with this file: k_snappy_decode hands LZ4 blocks to lz4_warp_decode, and k_lz4_compress shares
// the search above (snapc_next_match).
#include "lz4_kernels.cuh"
