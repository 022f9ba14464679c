// lz4_kernels.cuh — LZ4 blocks in and out: kLZ4Compression (trailer type 4) and, read only, kLZ4HCCompression (5).
//
// DocDB selects the block codec with its compression_type flag (docdb_rocksdb_util.cc:176-202). With format_version 2
// (compress_format_version 2, util/compression.h LZ4_Compress / LZ4_Uncompress) a stored LZ4 block is a varint32 of the
// uncompressed length followed by one raw LZ4 block (lz4_Block_format.md): sequences of a token (literal length << 4 |
// match length - 4; a nibble of 15 continues in extension bytes that each add their value, 255 meaning more follow),
// the literals, a 2-byte little-endian offset (1..65535) and the match length's extension bytes. The last sequence is
// literals only; the last 5 bytes of the block are literals and no match starts within its last 12 (the end-of-block
// rules LZ4_decompress_safe enforces). LZ4HC writes the same format with a stronger search.
//
// Input: the blocks go through snappy_kernels.cuh's sizes pass and warp-per-block decode together with raw and Snappy
// blocks; the decode kernel hands LZ4 blocks to lz4_warp_decode, which follows the Snappy decoder: every lane parses
// the tokens redundantly (uniform control flow), literal and match bytes are spread over the lanes, a match with an
// offset of at least 32 proceeds in rounds of 32 bytes and a closer one is a repeating pattern, and runs of 255-valued
// extension bytes are summed 32 bytes per ballot.
//
// Output: k_lz4_compress, one warp per assembled block into k_snappy_compress's scratch image, with its search
// (snapc_next_match: 32 positions per step, the same table, hash and match order) and an LZ4 emitter; k_snappy_gather
// then moves the stored forms. The encoder is the one written out beside host_sst.cc Lz4Compress, so that the
// host writer's index blocks and these data blocks come from one encoder.
//
// Included at the end of snappy_kernels.cuh, whose search and views it uses.
#pragma once

namespace ybgpu {

// Adds the extension bytes of a length whose nibble was 15, from src[*ip] on, to *len: each ballot looks at 32 bytes
// and finds the first that is not 255. False when the bytes run past the input or the length past any block.
__device__ __forceinline__ bool lz4_ext_len(const uint8_t* src, uint32_t size, uint32_t* ip, uint32_t* len, int lane) {
  const uint32_t FULL = 0xffffffffu;
  uint32_t stop, v;
  do {
    const uint32_t q = *ip + lane;
    v = q < size ? src[q] : 0u;
    stop = __ballot_sync(FULL, q >= size || v != 255u);
    if (!stop) { *ip += 32; *len += 255u * 32; }
  } while (!stop && *len < (1u << 30));                   // k_snappy_sizes admits no block this long
  const uint32_t k = stop ? static_cast<uint32_t>(__ffs(stop) - 1) : 0u;
  const uint32_t last = __shfl_sync(FULL, v, k);
  if (!stop || *ip + k >= size) return false;
  *len += 255u * k + last;
  *ip += k + 1;
  return true;
}

// One LZ4 block by one warp: the stream src[ip, size) (ip: behind the varint32 preamble) into dst[0, ulen).
__device__ __forceinline__ bool lz4_warp_decode(const uint8_t* src, uint32_t size, uint32_t ip, uint8_t* dst, uint32_t ulen, int lane) {
  uint32_t op = 0;
  bool bad = false;
  for (;;) {
    if (ip >= size) { bad = true; break; }                // truncated token
    const uint32_t token = src[ip++];
    uint32_t lit = token >> 4;
    if (lit == 15 && !lz4_ext_len(src, size, &ip, &lit, lane)) { bad = true; break; }
    if (size - ip < lit || ulen - op < lit) { bad = true; break; }
    for (uint32_t i = lane; i < lit; i += 32) dst[op + i] = src[ip + i];
    ip += lit; op += lit;
    if (ip == size) break;                                // the last sequence: literals only
    if (ulen - op < 12 || size - ip < 2) { bad = true; break; }   // a match within the last 12 bytes, or a truncated offset
    const uint32_t off = src[ip] | (static_cast<uint32_t>(src[ip + 1]) << 8);
    ip += 2;
    uint32_t len = token & 15;
    if (len == 15 && !lz4_ext_len(src, size, &ip, &len, lane)) { bad = true; break; }
    len += 4;
    if (off == 0 || off > op || ulen - op < len + 5) { bad = true; break; }   // the last 5 bytes are literals
    __syncwarp();                                         // what earlier sequences wrote is visible to every lane
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
  return !bad && op == ulen;
}

// One sequence at out + *op: the literals in[from, to) and, unless mlen is 0 (the closing sequence), a match of mlen
// bytes at offset off. Extension bytes are written by the lanes in parallel. False, with nothing written, when the
// output would reach limit.
__device__ __forceinline__ bool lz4_emit(uint8_t* out, uint32_t* op, uint32_t limit, const uint8_t* in, uint32_t from, uint32_t to,
                                         uint32_t mlen, uint32_t off, int lane) {
  const uint32_t L = to - from, M = mlen ? mlen - 4 : 0;
  const uint32_t nl = L >= 15 ? (L - 15) / 255 + 1 : 0;
  const uint32_t nm = M >= 15 ? (M - 15) / 255 + 1 : 0;
  const uint32_t total = 1 + nl + L + (mlen ? 2 + nm : 0);
  if (*op + total >= limit) return false;
  uint8_t* e = out + *op;
  if (lane == 0) e[0] = static_cast<uint8_t>((min(L, 15u) << 4) | min(M, 15u));
  for (uint32_t j = lane; j < nl; j += 32) e[1 + j] = static_cast<uint8_t>(j + 1 < nl ? 255u : (L - 15) % 255);
  warp_copy(e + 1 + nl, in + from, L, lane);
  if (mlen) {
    uint8_t* q = e + 1 + nl + L;
    if (lane < 2) q[lane] = static_cast<uint8_t>(off >> (8 * lane));
    for (uint32_t j = lane; j < nm; j += 32) q[2 + j] = static_cast<uint8_t>(j + 1 < nm ? 255u : (M - 15) % 255);
  }
  *op += total;
  return true;
}

// kLZ4Compression for every assembled block (same view, scratch image, 7/8 cutoff and outputs as k_snappy_compress).
__global__ void __launch_bounds__(SNAPC_WARPS * 32) k_lz4_compress(SnapCompView V) {
  __shared__ uint16_t s_pos[SNAPC_WARPS][1u << SNAPC_HASH_BITS];   // the hash table (snappy_kernels.cuh snapc_clear_table)
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
    bool give_up = n64 >= 0x7fffffffull;                  // kCompressionSizeLimit (block_based_table_builder.cc:642)
    uint32_t op = 0;
    if (!give_up) {                                       // varint32 preamble: the uncompressed length
      uint32_t v = n;
      while (v >= 128) { if (lane == 0) out[op] = static_cast<uint8_t>(v | 128); v >>= 7; op++; }
      if (lane == 0) out[op] = static_cast<uint8_t>(v);
      op++;
      if (op >= limit) give_up = true;
    }
    uint32_t lit = 0;                                     // block-absolute: literal runs span fragments
    for (uint32_t fs = 0; fs < n && !give_up; fs += SNAPC_FRAGMENT) {
      const uint8_t* f = in + fs;
      const uint32_t m = min(n - fs, SNAPC_FRAGMENT);
      const uint32_t smax = n - fs > 8 ? min(m, n - fs - 8) : 0u;   // positions p + 4 <= smax: p <= n - 12
      const uint32_t emax = n - fs > 5 ? min(m, n - fs - 5) : 0u;   // a match ends by n - 5
      snapc_clear_table(T, G, lane);
      uint32_t i = 0, mpos, c, len;
      SnapcBatch cur = snapc_prepare<0>(f, 0, smax, lane);
      while (snapc_next_match<0>(f, i, cur, smax, emax, T, G, lane, &mpos, &c, &len)) {
        if (!lz4_emit(out, &op, limit, in, lit, fs + mpos, len, mpos - c, lane)) { give_up = true; break; }
        lit = fs + mpos + len;
      }
    }
    if (!give_up && !lz4_emit(out, &op, limit, in, lit, n, 0, 0, lane)) give_up = true;   // the closing literals
    const bool keep = !give_up && op < limit;
    if (lane == 0) {
      if (keep) out[op] = 4;                              // the trailer's type byte: kLZ4Compression
      V.csize[b] = keep ? op : 0u;
      V.fsize[b] = (keep ? static_cast<unsigned long long>(op) : n64) + 5ull;
    }
  }
}

}  // namespace ybgpu
