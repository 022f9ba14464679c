// ingest_kernels.cuh — K0/K1 fused: one pass over the input files.
//
// Replaces, for shared-prefix inputs with internal keys of at most 64 bytes, the three passes
//   k_crc_blocks (ReadBlock checksum verification, table/format.cc:352-395),
//   k_prepass    (entry counts, validation; BlockIter walk, table/block.cc:348-447),
//   k_decode_*   (key reconstruction into fixed-stride records)
// by ONE kernel that reads every input byte from HBM exactly once:
//
//   * a data block (contents + 5-byte trailer) is staged into shared memory by one 1-D TMA bulk copy
//     (cp.async.bulk global->shared, completion on an mbarrier) — no register staging, no per-thread loads;
//   * lanes own restart intervals and walk the entry headers in shared memory (count + validation);
//   * one thread per entry computes the RAW CRC32C (zero initial register, no final complement) of the
//     entry's value and of the bytes in front of it (header + key delta). The block checksum is the GF(2)-
//     linear combination of the segment CRCs (crc(A || B) = crc(A) * x^(8|B|) + crc(B)), compared with the
//     stored trailer; the per-entry VALUE CRCs are kept (4 B per entry): the block encoder derives the
//     output blocks' checksums from them without ever looking at value bytes again (values are copied
//     verbatim from input to output, so their CRC contribution only needs shifting);
//   * the entry base of the block inside its file is known beforehand: the probe kernel counts a block's entries as
//     (restarts - 1) x restart interval + the entries of its last interval (only that interval's headers are walked,
//     ~1/7 of the block's sectors), a per-file scan turns the counts into bases (a decoupled look-back inside this
//     kernel was tried first: with ~450 blocks in flight every block ended up summing all in-flight predecessors);
//   * lanes walk their intervals a second time, rebuild the internal keys in registers and write records.
//
// CRC table look-ups dominate the kernel's instruction count (one per byte: there is no CRC / carry-less multiply
// instruction); the four 256-entry slicing tables are stored ING_REP = 8 times with the table index in the bank number,
// lane l uses copy l % 8 and rotates its look-up order by l / 8: no bank conflicts whatever the data (IngTab below).
//
// Anything this kernel does not take — other key encodings, keys longer than 64 bytes, blocks larger than the
// staging buffer, more than ING_MAXE entries in a block — raises J->ingest_fallback (not an error) and the host
// runs the general kernels (k_prepass, k_decode_all, k_crc_blocks, k_value_crc) instead.
//
// Included by engine.cu only (after encode_kernels.cuh: CRC tables and helpers).
#pragma once

namespace ybgpu {

constexpr int ING_CONSUMERS = 128;            // threads per consumer role: warps 0-3 rebuild keys and write records, warps 4-7 compute the CRCs
constexpr int ING_WALKER = 8, ING_PRODUCER = 9;   // warp 8: walker (entry headers), warp 9: producer (tickets, handles, bulk copies)
constexpr int ING_THREADS = 320;
constexpr uint32_t ING_BUF = 34304;           // staged bytes per block (33.5 KB): contents + trailer + alignment slack
constexpr int ING_MAXE = 512;                 // entries per block
constexpr int ING_REP = 8;                    // replication of the CRC tables
constexpr int ING_NVI = 4;                    // internal keys up to 64 bytes
constexpr int ING_BATCH = 8;                  // blocks claimed per ticket
constexpr int ING_FALLBACK_WIDER = 1;         // a key does not fit the guessed record stride: once more with the widest
constexpr int ING_FALLBACK_GENERAL = 2;       // not for this kernel: general path
constexpr size_t ING_SMEM = 2 * (ING_BUF + 32) + 4 * 256 * ING_REP * 4 + 2 * ING_MAXE * 12;

struct IngestView {
  const RunView* runs;
  const uint32_t* blk_base;        // [k+1] first global block index of every run
  uint32_t* ticket;
  const uint32_t* totals;          // [k] entries per run (the blocks' bases are run.blk_count[], an exclusive prefix)
  const RangeDev* range;           // nullptr = no key range
  int k, S, verify;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// 1-D TMA bulk copy global -> shared; dst, src 16-byte aligned, bytes a multiple of 16
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes),
               "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, %2;\n"      // suspended until the phase completes or the hint (ns) expires
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity), "r"(100000u)
      : "memory");
}

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }
// Per block: its entry count (in two parts, see below) and compression type; per run: the restart interval, read off
// the first block that has two intervals; a sample of key lengths.
__global__ void __launch_bounds__(256) k_restart_probe(const RunView* runs, const uint32_t* blk_base, int k, JobDev* J) {
  const uint32_t total = blk_base[k];
  for (uint32_t gb = blockIdx.x * blockDim.x + threadIdx.x; gb < total; gb += gridDim.x * blockDim.x) {
    int ri_ = 0;
    while (blk_base[ri_ + 1] <= gb) ri_++;
    const RunView& run = runs[ri_];
    const uint32_t b = gb - blk_base[ri_];
    const uint8_t* blk = run.data + run.blk_off[b];
    const uint32_t size = run.blk_size[b];
    uint32_t nres = size >= 4 ? ldg_u32_unaligned(blk + size - 4) : 0;
    const uint8_t type = blk[size];                        // trailer: compression type of the stored block
    if (type != 0) {
      // Snappy and LZ4 (LZ4HC) blocks are uncompressed by the host's next stage (snappy_kernels.cuh, lz4_kernels.cuh),
      // then the probe runs again
      if (type == 1 || type == 4 || type == 5) {
        atomicAdd(&J->n_compressed, 1u);
        if (type != 1) atomicAdd(&J->n_lz4, 1u);
      } else {
        dev_fail(J, DEV_ERR_COMPRESSED, b);
      }
      nres = 0;
    } else if (nres == 0 || static_cast<uint64_t>(nres) * 4 + 4 > size) { dev_fail(J, DEV_ERR_BAD_BLOCK, b); nres = 0; }
    if (nres == 0) continue;
    // entries of the block = (restarts - 1) full intervals + the last interval, whose headers are walked here
    {
      const uint32_t restarts_off = size - 4 - 4 * nres;
      uint32_t p = ldg_u32_unaligned(blk + restarts_off + 4 * (nres - 1));
      const uint32_t end = restarts_off;
      uint32_t n = 0, klen = 0;
      bool ok = p <= end;
      while (ok && p < end) {
        if (run.key_encoding == 2) {
          TspHeader th; uint32_t nk, ms, ml;
          const int h = parse_entry_header_tsp(blk + p, end - p, &th);
          ok = h && tsp_key_layout(th, klen, &nk, &ms, &ml);
          if (ok) { klen = nk; p += h + th.ns1 + th.ns2 + th.vlen; n++; }
        } else {
          uint32_t shared, non_shared, vlen;
          const int h = parse_entry_header(blk + p, end - p, &shared, &non_shared, &vlen);
          ok = h != 0;
          if (ok) { p += h + non_shared + vlen; n++; }
        }
      }
      if (!ok || p != end || n == 0 || n > 0xffff || nres - 1 > 0xffff) { dev_fail(J, DEV_ERR_BAD_ENTRY, b); n = 0; }
      run.blk_count[b] = ((nres - 1) << 16) | n;          // resolved by k_block_counts once the restart interval is known
    }
    // The first interval of a block with two intervals gives the restart interval; that of every 16th block is walked
    // as well: the longest key met is the host's guess for the record stride (a longer key inside k_ingest only costs a
    // second attempt with the widest stride).
    if ((nres >= 2 && __ldcg(&J->restart_interval[ri_]) == 0) || (nres >= 2 && (b & 15) == 0)) {
      // walk the first interval's headers (either encoding is delimited by the second restart offset)
      const uint32_t restarts_off = size - 4 - 4 * nres;
      uint32_t p = ldg_u32_unaligned(blk + restarts_off);
      const uint32_t end = ldg_u32_unaligned(blk + restarts_off + 4);
      if (p > end || end > restarts_off) { dev_fail(J, DEV_ERR_BAD_BLOCK, b); continue; }
      uint32_t n = 0, klen = 0, maxk = 0;
      bool ok = true;
      while (p < end && ok) {
        if (run.key_encoding == 2) {
          TspHeader th; uint32_t nk, ms, ml;
          const int h = parse_entry_header_tsp(blk + p, end - p, &th);
          ok = h && tsp_key_layout(th, klen, &nk, &ms, &ml);
          if (ok) { klen = nk; p += h + th.ns1 + th.ns2 + th.vlen; n++; }
        } else {
          uint32_t shared, non_shared, vlen;
          const int h = parse_entry_header(blk + p, end - p, &shared, &non_shared, &vlen);
          ok = h != 0;
          if (ok) { klen = shared + non_shared; p += h + non_shared + vlen; n++; }
        }
        maxk = max(maxk, klen);
      }
      if (!ok || p != end || n == 0) { dev_fail(J, DEV_ERR_BAD_ENTRY, b); continue; }
      atomicCAS(&J->restart_interval[ri_], 0u, n);
      atomicMax(&J->max_ikey_len, maxk);
    }
  }
}

// blk_count[b] = full intervals x restart interval + entries of the last interval (then scanned per file)
__global__ void __launch_bounds__(256) k_block_counts(const RunView* runs, const uint32_t* blk_base, int k, JobDev* J) {
  const uint32_t total = blk_base[k];
  for (uint32_t gb = blockIdx.x * blockDim.x + threadIdx.x; gb < total; gb += gridDim.x * blockDim.x) {
    int r = 0;
    while (blk_base[r + 1] <= gb) r++;
    const uint32_t b = gb - blk_base[r];
    const uint32_t v = runs[r].blk_count[b];
    runs[r].blk_count[b] = (v >> 16) * J->restart_interval[r] + (v & 0xffff);
  }
}

struct IngEntry { uint16_t estart, kstart, vstart, vlen, shared, klen; };    // offsets inside the block (a block is at most ING_BUF bytes), key delta geometry

// The four slicing tables, ING_REP = 8 copies, laid out so that the TABLE index is part of the bank number:
//   word address of T_t[e], copy c  =  e * 32 + t * 8 + c        (bank = t * 8 + c, independent of e)
// A lane uses copy (lane & 7) and looks the four bytes of a word step up in ROTATED order: in its k-th look-up it
// addresses table t = (k + (lane >> 3)) & 3. The 32 lanes of a warp then hit 32 different banks in every one of the
// four look-up instructions, whatever the data: no bank conflicts with 32 KB of tables.
struct IngTab {
  const uint32_t* base;            // table words in shared memory
  uint32_t sel[4];                 // PRMT selector extracting the byte table t_k consumes (T3 <-> byte 0 ... T0 <-> byte 3)
  uint32_t off[4];                 // t_k * 8 + copy
  uint32_t addr[4];                // shared-space byte address of word off[k] (a look-up is idx * 128 + addr[k]: one multiply-add)
  uint32_t copy;
};
__device__ __forceinline__ IngTab ing_tab_init(const uint32_t* base, uint32_t lane) {
  IngTab T;
  T.base = base; T.copy = lane & 7u;
#pragma unroll
  for (uint32_t k = 0; k < 4; k++) {
    const uint32_t t = (k + (lane >> 3)) & 3u;
    T.sel[k] = 0x4440u + (3u - t);
    T.off[k] = t * 8u + T.copy;
    T.addr[k] = static_cast<uint32_t>(__cvta_generic_to_shared(base)) + 4u * T.off[k];
  }
  return T;
}
// T0[x] (single byte steps: the lanes that share a copy collide — rare paths only)
__device__ __forceinline__ uint32_t ing_t0(const IngTab& T, uint32_t x) { return T.base[x * 32u + T.copy]; }
__device__ __forceinline__ uint32_t ing_crc_byte(const IngTab& T, uint32_t c, uint32_t byte) { return ing_t0(T, (c ^ byte) & 0xff) ^ (c >> 8); }
__device__ __forceinline__ uint32_t ing_crc_word(const IngTab& T, uint32_t c, uint32_t w) {
  c ^= w;
  uint32_t r = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    // address arithmetic in the shared window (the generic-pointer form costs an extra add of the window base per look-up)
    uint32_t v;
    asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(__byte_perm(c, 0u, T.sel[k]) * 128u + T.addr[k]));
    r ^= v;
  }
  return r;
}
// c * x^32 mod P (four zero bytes): what crc_clmul_reduce needs, as one conflict-free word step
__device__ __forceinline__ uint32_t ing_clmul_reduce(const IngTab& T, unsigned long long z) {
  z <<= 1;
  return ing_crc_word(T, static_cast<uint32_t>(z), 0u) ^ static_cast<uint32_t>(z >> 32);
}
// Raw CRC (zero initial register) of the shared-memory bytes [p, p + n). The word grid is aligned to the END of the
// span: the first word may reach up to 3 bytes in front of p, which are masked to zero (leading zeros do not move a
// zero register) — so there are only whole-word steps, no byte steps at either end. Every word is one aligned load
// plus a funnel shift with its predecessor. Touches up to 6 bytes in front of p and 3 behind the span.
// `c_in` = register to continue from (only zero keeps the leading-zero argument: callers pass 0 for a fresh span).
__device__ __forceinline__ uint32_t ing_crc_words(const IngTab& T, const uint32_t* wb, uint32_t bits, uint32_t nw, uint32_t first_mask) {
  uint32_t c = 0;
  uint32_t prev = wb[0];
  for (uint32_t i = 0; i < nw; i++) {
    const uint32_t cur = wb[i + 1];
    uint32_t w = __funnelshift_r(prev, cur, bits);
    if (i == 0) w &= first_mask;
    c = ing_crc_word(T, c, w);
    prev = cur;
  }
  return c;
}
__device__ __forceinline__ uint32_t ing_crc_span(const IngTab& T, const uint8_t* p, uint32_t n) {
  if (n == 0) return 0;
  const uint8_t* end = p + n;
  const uint32_t a = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(end) & 3);
  const uint32_t nw = (n + 3) >> 2, lead = 4 * nw - n;
  const uint32_t* wb = reinterpret_cast<const uint32_t*>(end - 4 * nw - a);
  return ing_crc_words(T, wb, 8 * a, nw, 0xffffffffu << (8 * lead));
}
// The same with two independent chains over the two halves of a long span (the look-up latency of one chain no longer
// bounds a thread), joined by one multiplication.
__device__ __forceinline__ uint32_t ing_crc_span2(const IngTab& T, const uint8_t* p, uint32_t n) {
  if (n < 96) return ing_crc_span(T, p, n);
  const uint8_t* end = p + n;
  const uint32_t a = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(end) & 3), bits = 8 * a;
  const uint32_t nw = (n + 3) >> 2, lead = 4 * nw - n;
  const uint32_t* wb = reinterpret_cast<const uint32_t*>(end - 4 * nw - a);
  const uint32_t h = nw >> 1, h2 = nw - h;          // first chain: words [0, h), second: [h, nw); h <= h2 <= h + 1
  uint32_t c = 0, d = 0;
  uint32_t pc = wb[0], pd = wb[h];
  const uint32_t first_mask = 0xffffffffu << (8 * lead);
  for (uint32_t i = 0; i < h; i++) {
    const uint32_t cc = wb[i + 1], cd = wb[h + i + 1];
    uint32_t x = __funnelshift_r(pc, cc, bits);
    const uint32_t y = __funnelshift_r(pd, cd, bits);
    if (i == 0) x &= first_mask;
    c = ing_crc_word(T, c, x);
    d = ing_crc_word(T, d, y);
    pc = cc; pd = cd;
  }
  if (h2 > h) d = ing_crc_word(T, d, __funnelshift_r(pd, wb[nw], bits));
  return ing_clmul_reduce(T, crc_clmul(c, __ldg(&g_crc_xpow8[4 * h2]))) ^ d;
}

// What the producer resolves for a block before it requests the block's bytes.
struct IngBlk {
  const uint8_t* gsrc;             // 16-byte aligned start of the bulk copy (mis bytes in front of the block)
  unsigned long long boff;         // block offset inside the data file
  uint8_t* rec; uint64_t* val_off; uint32_t* val_crc;
  unsigned long long ht_filter;
  uint32_t run, b, size, mis, span;
  uint32_t base, expect;           // first entry of the block inside its file, entries in the block (probe + scan)
  uint32_t ri;                     // restart interval of the file (0xffffffff: every block has one interval)
  uint32_t valid;                  // 0: past the end, 1: staged, 2: not for this kernel (skipped)
};

// Warp-specialised: nothing a block needs from global memory is fetched by the threads that work on it.
//   warp 5 (producer): claims ING_BATCH consecutive blocks per atomic, resolves their handles, entry bases and output
//     pointers (lanes in parallel), and issues one bulk copy per block into a free staging buffer;
//   warp 4 (walker): parses the entry headers of a staged block — the only serial part, an entry's position
//     depends on its predecessors' lengths; lanes own restart intervals — into the entry table, validates, and
//     computes the CRC of the block's tail;
//   warps 0-3 (consumers): one thread per entry — internal key (own delta + inherited prefix bytes), record, value
//     CRC, the entry's share of the block checksum.
// Stages hand over through mbarriers (full -> walked -> empty), so the walker works on block i + 1 and the bulk
// copy of block i + 2 is in flight while the consumers are on block i; the consumers never meet a CTA-wide barrier.
__global__ void __launch_bounds__(ING_THREADS, 2) k_ingest(IngestView V, JobDev* J) {
  extern __shared__ __align__(16) uint8_t ing_smem[];
  // two staging buffers (16 B front pad: key deltas are fetched with up to 15 + 3 bytes in front; 16 B back pad),
  // the CRC tables, two entry tables
  uint8_t* const buf0 = ing_smem + 16;
  uint32_t* tabs = reinterpret_cast<uint32_t*>(ing_smem + 2 * (ING_BUF + 32));        // 4 * 256 * ING_REP words
  IngEntry* const etab0 = reinterpret_cast<IngEntry*>(tabs + 4 * 256 * ING_REP);      // 2 * ING_MAXE
  __shared__ __align__(8) unsigned long long full_bar[2], walked_bar[2], empty_bar[2];
  __shared__ IngBlk sh_blk[2];                   // per stage: the block staged there
  __shared__ IngBlk sh_batch[ING_BATCH];         // claimed, not yet requested
  __shared__ uint32_t sh_nent[2], sh_tail[2], sh_acc[2], sh_cnt[2];
  __shared__ uint4 sh_upto[17];                  // sh_upto[n]: 0xff in the first n bytes of a 16-byte vector
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) {
    const uint32_t v = (&g_crc_tab[0][0])[i];        // i = t * 256 + e
    const uint32_t t = static_cast<uint32_t>(i) >> 8, e = static_cast<uint32_t>(i) & 255u;
#pragma unroll
    for (int c = 0; c < ING_REP; c++) tabs[e * 32u + t * 8u + c] = v;
  }
  const IngTab T = ing_tab_init(tabs, static_cast<uint32_t>(lane));
  if (threadIdx.x < 17) sh_upto[threadIdx.x] = low_bytes_mask16(static_cast<int>(threadIdx.x));
  if (threadIdx.x == 0) {
    for (int s = 0; s < 2; s++) {
      mbar_init(&full_bar[s], 1); mbar_init(&walked_bar[s], 1); mbar_init(&empty_bar[s], 2 * ING_CONSUMERS / 32);
      sh_acc[s] = 0; sh_cnt[s] = 0;
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const uint32_t total_blocks = V.blk_base[V.k];
  const int S = V.S;

  if (wid == ING_PRODUCER) {
    // ---------------- producer
    uint32_t uses[2] = {0, 0};
    int stage = 0;
    bool more = true;
    while (more) {
      uint32_t g0 = 0;
      if (lane == 0) g0 = atomicAdd(V.ticket, static_cast<uint32_t>(ING_BATCH));
      g0 = __shfl_sync(0xffffffffu, g0, 0);
      if (lane < ING_BATCH) {
        IngBlk x;
        x.valid = 0;
        const uint32_t gb = g0 + lane;
        if (gb < total_blocks) {
          int r = 0;
          while (V.blk_base[r + 1] <= gb) r++;
          const RunView& run = V.runs[r];
          x.run = static_cast<uint32_t>(r); x.b = gb - V.blk_base[r];
          x.boff = run.blk_off[x.b]; x.size = run.blk_size[x.b];
          const uint8_t* g = run.data + x.boff;
          x.mis = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(g) & 15);
          x.gsrc = g - x.mis;
          x.span = (x.mis + x.size + 5 + 15) & ~15u;
          x.rec = run.rec; x.val_off = run.val_off; x.val_crc = run.val_crc; x.ht_filter = run.ht_filter;
          x.base = run.blk_count[x.b];
          x.expect = ((x.b + 1 < run.nb) ? run.blk_count[x.b + 1] : V.totals[r]) - x.base;
          const uint32_t ri = J->restart_interval[r];
          x.ri = ri ? ri : 0xffffffffu;
          x.valid = 1;
          // not for this kernel (the host switches to the general path): nothing to stage
          if (x.span > ING_BUF || run.key_encoding != 1) { atomicMax(&J->ingest_fallback, ING_FALLBACK_GENERAL); x.valid = 2; }
        }
        sh_batch[lane] = x;
      }
      __syncwarp();
      if (lane == 0) {
        for (int n = 0; n < ING_BATCH; n++) {
          const uint32_t v = sh_batch[n].valid;
          if (v == 0) { more = false; break; }
          if (v == 2) continue;
          if (uses[stage]) mbar_wait(&empty_bar[stage], (uses[stage] - 1) & 1);      // the consumers are done with its previous block
          uses[stage]++;
          sh_blk[stage] = sh_batch[n];
          mbar_expect_tx(&full_bar[stage], sh_batch[n].span);
          bulk_g2s(buf0 + stage * (ING_BUF + 32), sh_batch[n].gsrc, sh_batch[n].span, &full_bar[stage]);
          stage ^= 1;
        }
        if (g0 + ING_BATCH >= total_blocks) more = false;
      }
      more = __shfl_sync(0xffffffffu, more ? 1 : 0, 0) != 0;
      stage = __shfl_sync(0xffffffffu, stage, 0);
    }
    if (lane == 0) {                               // end marker for the walker and, through it, the consumers
      if (uses[stage]) mbar_wait(&empty_bar[stage], (uses[stage] - 1) & 1);
      sh_blk[stage].valid = 0;
      mbar_arrive(&full_bar[stage]);
    }
    return;
  }

  if (wid == ING_WALKER) {
    // ---------------- walker
    uint32_t maxk = 0;
    for (uint32_t it = 0;; it++) {
      const int stage = it & 1;
      mbar_wait(&full_bar[stage], (it >> 1) & 1);
      const uint32_t valid = sh_blk[stage].valid;
      if (!valid) {
        if (lane == 0) { sh_nent[stage] = 0xffffffffu; mbar_arrive(&walked_bar[stage]); }
        break;
      }
      const uint32_t size = sh_blk[stage].size, b = sh_blk[stage].b, ri = sh_blk[stage].ri, expect = sh_blk[stage].expect;
      const uint8_t* blk = buf0 + stage * (ING_BUF + 32) + sh_blk[stage].mis;
      IngEntry* etab = etab0 + stage * ING_MAXE;
      const uint32_t nres = ld_u32_unaligned(blk + size - 4);
      uint32_t bad = 0;
      if (nres == 0 || static_cast<uint64_t>(nres) * 4 + 4 > size) bad = DEV_ERR_BAD_BLOCK;
      else if (blk[size] != 0) bad = DEV_ERR_COMPRESSED;
      const uint32_t restarts_off = bad ? 0 : size - 4 - 4 * nres;
      uint32_t my_n = 0;
      int fallback = 0;
      if (!bad) {
        for (uint32_t r = lane; r < nres; r += 32) {
          uint32_t p = ld_u32_unaligned(blk + restarts_off + 4 * r);
          const uint32_t end = (r + 1 < nres) ? ld_u32_unaligned(blk + restarts_off + 4 * (r + 1)) : restarts_off;
          if (p > end || end > restarts_off) { bad = DEV_ERR_BAD_BLOCK; break; }
          uint32_t n = 0, klen = 0;
          const uint64_t slot0 = static_cast<uint64_t>(r) * (ri == 0xffffffffu ? 0u : ri);
          while (p < end) {
            uint32_t shared, non_shared, vlen;
            const int h = parse_entry_header(blk + p, end - p, &shared, &non_shared, &vlen);
            if (!h || shared > klen || (n == 0 && shared != 0) || static_cast<uint64_t>(p) + h + non_shared + vlen > end) { bad = DEV_ERR_BAD_ENTRY; break; }
            klen = shared + non_shared;
            if (klen < 8) { bad = DEV_ERR_SHORT_KEY; break; }
            maxk = max(maxk, klen);
            const uint64_t slot = slot0 + n;
            if (slot >= ING_MAXE || klen > 16 * ING_NVI) { fallback = ING_FALLBACK_GENERAL; break; }
            if (klen > static_cast<uint32_t>(S) - 8) fallback = ING_FALLBACK_WIDER;      // user key longer than S - 16: the walk goes on (longest key)
            IngEntry e;
            e.estart = static_cast<uint16_t>(p); e.kstart = static_cast<uint16_t>(p + h); e.vstart = static_cast<uint16_t>(p + h + non_shared);
            e.vlen = static_cast<uint16_t>(vlen); e.shared = static_cast<uint16_t>(shared); e.klen = static_cast<uint16_t>(klen);
            etab[slot] = e;
            p += h + non_shared + vlen;
            n++;
          }
          if (bad || fallback == ING_FALLBACK_GENERAL) break;
          // every interval but the last of a block is full (BlockBuilder restarts every block_restart_interval entries)
          if (r + 1 < nres) { if (n != ri) { bad = DEV_ERR_IRREGULAR_RESTARTS; break; } }
          else if (n > ri || n == 0) { bad = n ? DEV_ERR_IRREGULAR_RESTARTS : DEV_ERR_BAD_ENTRY; break; }
          my_n += n;
        }
      }
      bad = __reduce_max_sync(0xffffffffu, bad);
      fallback = static_cast<int>(__reduce_max_sync(0xffffffffu, static_cast<uint32_t>(fallback)));
      uint32_t n_ent = __reduce_add_sync(0xffffffffu, my_n);
      uint32_t tail = 0;
      if (lane == 0) {
        if (bad) dev_fail(J, bad, b);
        if (fallback) atomicMax(&J->ingest_fallback, fallback);
        if (bad || fallback) n_ent = 0;
        // the block's entry count was fixed by the probe + scan; it must agree with what the walk found
        else if (n_ent != expect) { dev_fail(J, DEV_ERR_IRREGULAR_RESTARTS, b); n_ent = 0; }
        // (the CRC of the block's tail is left to the CRC warps: this warp is the serial stage of the pipeline — a lane
        // parses its restart interval entry by entry — and what it does beyond that lengthens the pipeline period.)
        sh_nent[stage] = n_ent; sh_tail[stage] = tail;
      }
      __syncwarp();                                // the lanes' entry table writes are ordered before lane 0's arrive
      if (lane == 0) mbar_arrive(&walked_bar[stage]);
    }
    maxk = __reduce_max_sync(0xffffffffu, maxk);
    if (lane == 0 && maxk > __ldcg(&J->max_ikey_len)) atomicMax(&J->max_ikey_len, maxk);
    return;
  }

  // ---------------- consumers
  const bool ranged = V.range != nullptr;
  for (uint32_t it = 0;; it++) {
    const int stage = it & 1;
    mbar_wait(&walked_bar[stage], (it >> 1) & 1);
    const uint32_t n_ent = sh_nent[stage];
    if (n_ent == 0xffffffffu) break;
    const IngBlk& cur = sh_blk[stage];
    const uint32_t size = cur.size, base = cur.base;
    const uint64_t boff = cur.boff;
    const unsigned long long ht_filter = cur.ht_filter;
    uint8_t* const rec0 = cur.rec;
    uint64_t* const val_off = cur.val_off;
    uint32_t* const val_crc = cur.val_crc;
    const uint8_t* blk = buf0 + stage * (ING_BUF + 32) + cur.mis;
    const IngEntry* etab = etab0 + stage * ING_MAXE;
    const uint32_t L = size + 1;                       // contents + type byte
    const RunView& crun = V.runs[cur.run];
    const uint32_t cf_n = crun.cf_n;
    const bool filtered = ht_filter != 0xfffffffffffffffeull || ranged || cf_n != 0;
    unsigned long long acc = 0;                        // XOR of unreduced carry-less products (CRC warps)
    const uint32_t rt = threadIdx.x & (ING_CONSUMERS - 1);   // thread index inside its role
    if (wid < ING_CONSUMERS / 32) {
    for (uint32_t e = rt; e < n_ent; e += ING_CONSUMERS) {
      const IngEntry en = etab[e];
      uint4 kv[ING_NVI];
#pragma unroll
      for (int w = 0; w < ING_NVI; w++) kv[w] = make_uint4(0, 0, 0, 0);
      // 16 delta bytes for key offsets [16 w, 16 w + 16) of an entry whose delta starts at key offset a (its `shared`):
      // any alignment, shared memory; up to 15 + 3 bytes in front of the delta are touched
      auto fetch = [&](uint32_t kstart, uint32_t a, int w) {
        const uint8_t* src = blk + kstart + 16 * w - static_cast<int>(a);
        const uint32_t sh = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(src) & 3);
        const uint32_t* sa = reinterpret_cast<const uint32_t*>(src - sh);
        const uint32_t w0 = sa[0], w1 = sa[1], w2 = sa[2], w3 = sa[3], w4 = sa[4];
        const uint32_t bits = sh * 8;
        return make_uint4(__funnelshift_r(w0, w1, bits), __funnelshift_r(w1, w2, bits), __funnelshift_r(w2, w3, bits), __funnelshift_r(w3, w4, bits));
      };
      // own delta: key bytes [shared, klen). Bytes in front of `shared` inside its first window are overwritten below,
      // bytes behind klen are never looked at (the record write masks by the key length)
#pragma unroll
      for (int w = 0; w < ING_NVI; w++)
        if (16 * w + 16 > static_cast<int>(en.shared) && 16 * w < static_cast<int>(en.klen)) kv[w] = fetch(en.kstart, en.shared, w);
      // inherited bytes [0, shared): walking back, an entry contributes the bytes between its own `shared` and the
      // lowest `shared` met so far (the restart entry has shared = 0 and ends the walk; the walker validated all
      // that). A contribution overwrites everything below `need` in its windows: what it writes below its own
      // `shared` is overwritten in turn by the entries further back.
      {
        uint32_t need = en.shared;
        for (uint32_t j = e; need; ) {
          j--;
          const uint32_t sj = etab[j].shared;
          if (sj < need) {
            const uint32_t kstart = etab[j].kstart;
#pragma unroll
            for (int w = 0; w < ING_NVI; w++) {
              if (16 * w + 16 <= static_cast<int>(sj) || 16 * w >= static_cast<int>(need)) continue;
              const uint4 nw = fetch(kstart, sj, w);
              const uint4 m = sh_upto[min(need - 16 * w, 16u)];
              kv[w].x = (nw.x & m.x) | (kv[w].x & ~m.x);
              kv[w].y = (nw.y & m.y) | (kv[w].y & ~m.y);
              kv[w].z = (nw.z & m.z) | (kv[w].z & ~m.z);
              kv[w].w = (nw.w & m.w) | (kv[w].w & ~m.w);
            }
            need = sj;
          }
        }
      }
      const uint32_t klen = en.klen, ulen = klen - 8, vlen = en.vlen;
      // suffix = internal-key bytes [ulen, ulen + 8)
      uint4 va = kv[0], vb = kv[1];
#pragma unroll
      for (int w = 1; w < ING_NVI; w++) if (static_cast<int>(ulen >> 4) == w) { va = kv[w]; vb = (w + 1 < ING_NVI) ? kv[w + 1] : make_uint4(0, 0, 0, 0); }
      uint32_t s0, s1;
      {
        uint32_t w0 = va.x, w1 = va.y, w2 = va.z, w3 = va.w, w4 = vb.x, w5 = vb.y;
        const uint32_t sh = ulen & 15, qq = sh >> 2, bits = (sh & 3) * 8;
        if (qq & 1) { w0 = w1; w1 = w2; w2 = w3; w3 = w4; w4 = w5; }
        if (qq & 2) { w0 = w2; w1 = w3; w2 = w4; }
        s0 = __funnelshift_r(w0, w1, bits); s1 = __funnelshift_r(w1, w2, bits);
      }
      uint8_t flags = 0;
      if (filtered) {
        // rare: per-file HybridTime filter / key range of a subcompaction — the user key as bytes
        __align__(16) uint8_t kb[16 * ING_NVI];
#pragma unroll
        for (int w = 0; w < ING_NVI; w++) reinterpret_cast<uint4*>(kb)[w] = kv[w];
        if ((ht_filter != HT_FILTER_NONE || cf_n) && hidden_by_ht_filters(kb, ulen, ht_filter, crun.cf_oid, crun.cf_ht, cf_n)) flags |= REC_F_HT_FILTERED;
        if (ranged) {
          if (V.range->lower_len && cmp_raw(kb, ulen, V.range->lower, V.range->lower_len) < 0) flags |= REC_F_OUT_OF_RANGE;
          if (V.range->upper_len && cmp_raw(kb, ulen, V.range->upper, V.range->upper_len) >= 0) flags |= REC_F_OUT_OF_RANGE;
        }
      }
      uint8_t* rec = rec0 + static_cast<size_t>(base + e) * S;
      const int key_vecs = (S - 16) >> 4;
#pragma unroll
      for (int w = 0; w < ING_NVI; w++) {
        if (w < key_vecs) {
          const uint4 m = sh_upto[min(max(static_cast<int>(ulen) - 16 * w, 0), 16)];
          reinterpret_cast<uint4*>(rec)[w] = make_uint4(kv[w].x & m.x, kv[w].y & m.y, kv[w].z & m.z, kv[w].w & m.w);
        }
      }
      const uint8_t vfirst = vlen ? blk[en.vstart] : 0;
      uint4 tr;
      tr.x = s0; tr.y = s1;
      tr.z = ulen | (static_cast<uint32_t>(vfirst) << 16) | (static_cast<uint32_t>(flags) << 24);
      tr.w = vlen;
      *reinterpret_cast<uint4*>(rec + S - 16) = tr;
      val_off[base + e] = boff + en.vstart;
    }
    } else {
    for (uint32_t e = rt; e < n_ent; e += ING_CONSUMERS) {
      const IngEntry en = etab[e];
      const uint32_t vlen = en.vlen;
      // CRCs
      const uint32_t vc = ing_crc_span2(T, blk + en.vstart, vlen);
      val_crc[base + e] = vc;
      if (V.verify) {
        const uint32_t gc = ing_crc_span(T, blk + en.estart, en.vstart - en.estart);
        // gap * x^(8 (bytes behind the gap)) + value * x^(8 (bytes behind the value)), unreduced (L < 64 K: inside the table)
        acc ^= crc_clmul(gc, __ldg(&g_crc_xpow8[L - en.vstart])) ^ crc_clmul(vc, __ldg(&g_crc_xpow8[L - en.vstart - vlen]));
      }
    }
    }
    if (wid >= ING_CONSUMERS / 32 && V.verify && n_ent) {
      uint32_t a32 = ing_clmul_reduce(T, acc);
      if (rt == ING_CONSUMERS - 1) {
        // tail: restart array, restart count, type byte; and the 0xffffffff initial register's share (L < 64 K)
        const uint32_t nres = ld_u32_unaligned(blk + size - 4);
        const uint32_t restarts_off = size - 4 - 4 * nres;
        a32 ^= ing_crc_span(T, blk + restarts_off, L - restarts_off) ^ ing_clmul_reduce(T, crc_clmul(__ldg(&g_crc_xpow8[L]), 0xffffffffu));
      }
      a32 = __reduce_xor_sync(0xffffffffu, a32);
      if (lane == 0) {
        if (a32) atomicXor(&sh_acc[stage], a32);
        __threadfence_block();
        if (atomicAdd(&sh_cnt[stage], 1u) == ING_CONSUMERS / 32 - 1) {
          // the last warp of the block: entries + tail + initial register, final complement, against the trailer
          __threadfence_block();
          const uint32_t r = atomicExch(&sh_acc[stage], 0u) ^ sh_tail[stage];
          sh_cnt[stage] = 0;
          if (crc_mask(~r) != ld_u32_unaligned(blk + size + 1)) dev_fail(J, DEV_ERR_BAD_CRC, cur.b);
        }
      }
    }
    __syncwarp();                                  // every lane's reads of the stage are done before lane 0 releases it
    if (lane == 0) mbar_arrive(&empty_bar[stage]);
  }
}

// General path: RAW CRC32C of every value, one thread per entry, straight from the data file in HBM.
__global__ void __launch_bounds__(256) k_value_crc(const RunView* runs, int k, int S) {
  __shared__ uint32_t tabs[4 * 256 * ING_REP];
  for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) {
    const uint32_t v = (&g_crc_tab[0][0])[i];
#pragma unroll
    for (int c = 0; c < ING_REP; c++) tabs[i * ING_REP + c] = v;
  }
  __syncthreads();
  const uint32_t copy = threadIdx.x & (ING_REP - 1);
  for (int r = 0; r < k; r++) {
    const RunView& run = runs[r];
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < run.n_entries; i += gridDim.x * blockDim.x) {
      const uint8_t* rec = run.rec + static_cast<size_t>(i) * S;
      uint32_t n = rec_vlen(rec, S);
      const uint8_t* p = run.data + run.val_off[i];
      uint32_t c = 0;
      while (n && (reinterpret_cast<uintptr_t>(p) & 3)) { c = tabs[(((c ^ __ldg(p)) & 0xff)) * ING_REP + copy] ^ (c >> 8); p++; n--; }
      const uint32_t* w = reinterpret_cast<const uint32_t*>(p);
      for (uint32_t q = 0; q < (n >> 2); q++) {
        c ^= __ldg(w + q);
        c = tabs[((3 << 8) + (c & 0xff)) * ING_REP + copy] ^ tabs[((2 << 8) + ((c >> 8) & 0xff)) * ING_REP + copy] ^
            tabs[((1 << 8) + ((c >> 16) & 0xff)) * ING_REP + copy] ^ tabs[(c >> 24) * ING_REP + copy];
      }
      p += n & ~3u;
      for (uint32_t q = 0; q < (n & 3); q++) c = tabs[(((c ^ __ldg(p + q)) & 0xff)) * ING_REP + copy] ^ (c >> 8);
      run.val_crc[i] = c;
    }
  }
}

}  // namespace ybgpu
