// encode_kernels.cuh — K5: the output side of the compaction on the GPU.
//
// Turns the surviving entries (dense, in output order) into the data file of a split SST exactly
// as rocksdb::BlockBasedTableBuilder would (table/block_based_table_builder.cc:498-707):
//   * BlockBuilder entry encoding, restart every `ri` entries (table/block_builder.cc:347-412);
//   * FlushBlockBySizePolicy block cuts (table/flush_block_policy.cc:45-76) — a sequential rule
//     (each cut depends on where the block started), resolved in parallel by computing, for every
//     entry s, next[s] = first entry of the following block if a block started at s, and then
//     following that chain with two levels of segment "exit" tables;
//   * 5-byte trailers with masked CRC32C over block + type (:669-698), CRC computed by a
//     warp-parallel slicing-by-4 kernel combined with GF(2) shifts (also used to verify inputs).
//
// Included by engine.cu only.
#pragma once

namespace ybgpu {

constexpr int SEG = 4096;          // entries per chain segment
constexpr int GROUP_SEGS = 64;     // segments per group

struct EncView {
  const RunView* runs;
  const Desc* kept;                // dense survivors [n]
  const ValueRewrite* rewrites;
  uint32_t* nr;                    // [n] encoded size of entry as a non-restart entry
  uint16_t* shared;                // [n] bytes shared with the previous survivor's internal key
  int16_t* D;                      // [n] size difference if the entry is a restart point (negative values possible with
                                   //     three_shared_parts; all sums below are modulo 2^64, differences come out right)
  unsigned long long* P;           // [n+1] exclusive prefix of nr
  unsigned long long* QQ;          // [n] inclusive prefix of D within the entry's residue class mod ri
  uint32_t* next;                  // [n]
  uint32_t* exit1;                 // [n] first chain element >= end of s's segment
  uint32_t n;
  uint32_t ri;                     // block_restart_interval
  uint32_t ri_shift;               // log2(ri)
  uint32_t block_size;
  uint32_t deviation;
  uint32_t guess;                  // ~0.85 x expected entries per block: first probe of k_next's galloping search
  int key_encoding;                // 1 = shared_prefix, 2 = three_shared_parts (rocksdb/types.h:50-56)
  uint16_t* fk_len;                // [n] bloom filter key length of the entry (0 = none), nullptr = no filter policy
  const uint16_t* fk_src;          // [N] the same by input entry id, written by the merge kernel's DocKey walk
  const uint32_t* fkh_src;         // [N] bloom hash of the filter key by input entry id (merge kernel), or nullptr
  uint32_t* max_add;               // [1] largest size-estimate increment of one entry (FlushBlockBySizePolicy's `estimated size after`)
};

__device__ __forceinline__ uint64_t umin64(uint64_t a, uint64_t b) { return a < b ? a : b; }
__device__ __forceinline__ uint32_t varint_len(uint32_t v) { return v < (1u << 7) ? 1 : v < (1u << 14) ? 2 : v < (1u << 21) ? 3 : v < (1u << 28) ? 4 : 5; }

// Compact the merged-order descriptors into the dense survivor list. Every warp owns a contiguous
// slice of the chunk and walks it 32 descriptors at a time (coalesced 16-byte loads); positions
// come from ballots, the warp bases from a count pass over the same (cache-resident) slice.
__global__ void __launch_bounds__(EMIT_THREADS) k_compact_desc(const Desc* desc, uint64_t N, const Sums3* partial, Desc* kept) {
  constexpr int NW = EMIT_THREADS / 32, PER_WARP = EMIT_CHUNK / NW;
  static_assert(sizeof(Desc) == 16 && PER_WARP % 32 == 0, "descriptor layout");
  __shared__ uint32_t wcount[NW];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint64_t base = static_cast<uint64_t>(blockIdx.x) * EMIT_CHUNK + static_cast<uint64_t>(wid) * PER_WARP;
  const uint4* dv = reinterpret_cast<const uint4*>(desc);
  uint32_t cnt = 0;
  for (int r = 0; r < PER_WARP; r += 32) {
    const uint64_t i = base + r + lane;
    // flags live in byte 2 of the third word (gid, vlen_out, klen | flags << 16 | run << 24, rewrite_slot)
    const bool keep = i < N && ((__ldg(reinterpret_cast<const uint32_t*>(desc + i) + 2) >> 16) & ENT_KEEP);
    cnt += __popc(__ballot_sync(0xffffffffu, keep));
  }
  if (lane == 0) wcount[wid] = cnt;
  __syncthreads();
  uint64_t o = partial[blockIdx.x].n;
  for (int w = 0; w < wid; w++) o += wcount[w];
  for (int r = 0; r < PER_WARP; r += 32) {
    const uint64_t i = base + r + lane;
    uint4 d = make_uint4(0, 0, 0, 0);
    if (i < N) d = __ldg(dv + i);
    const bool keep = ((d.z >> 16) & ENT_KEEP) != 0;
    const uint32_t m = __ballot_sync(0xffffffffu, keep);
    if (keep) reinterpret_cast<uint4*>(kept)[o + __popc(m & ((1u << lane) - 1))] = d;
    o += __popc(m);
  }
}

__device__ __forceinline__ const uint8_t* kept_rec(const EncView& E, const Desc& d, int S) {
  const RunView& run = E.runs[d.run];
  return run.rec + static_cast<size_t>(d.gid - run.gid_base) * S;
}

// Internal-key byte i of a survivor (user key bytes, then the 8-byte suffix, zeroed seq if flagged).
__device__ __forceinline__ uint64_t kept_suffix(const uint8_t* rec, const Desc& d, int S) {
  uint64_t s = rec_suffix(rec, S);
  return (d.flags & ENT_ZERO_SEQ) ? (s & 0xff) : s;
}

// Per survivor: shared prefix with the previous survivor's internal key, encoded size as a non-restart entry (nr) and as
// a restart point (rs). Returns the most the entry can add to FlushBlockBySizePolicy's estimate.
__device__ __forceinline__ uint32_t entry_sizes(const EncView& E, int S, uint32_t j, const Desc& d, uint32_t* nr_out, uint32_t* rs_out, uint32_t* shared_out) {
  const uint32_t klen = d.klen, ulen = klen - 8u, vlen = d.vlen_out;
  const uint32_t add = klen + vlen + 8u + varint_len(klen) + varint_len(vlen);
  // the merge kernel has usually compared the key with the previous survivor's already (see its phase (e))
  if (E.key_encoding != 2 && j > 0 && !(d.flags & ENT_VAL_REENCODE) && (d.rewrite_slot & 0xffffu) != 0xffffu) {
    const uint32_t shared = d.rewrite_slot & 0xffffu;
    *nr_out = varint_len(shared) + varint_len(klen - shared) + varint_len(vlen) + (klen - shared) + vlen;
    *rs_out = 1 + varint_len(klen) + varint_len(vlen) + klen + vlen;
    *shared_out = shared;
    return add;
  }
  const uint8_t* rec = kept_rec(E, d, S);
  uint32_t shared = 0;
  if (j > 0) {
    const Desc pd = E.kept[j - 1];
    const uint8_t* prec = kept_rec(E, pd, S);
    const uint32_t pul = pd.klen - 8u;
    const uint32_t m = min(ulen, pul);
    shared = common_prefix_len(rec, m, prec, m);
    if (shared == m) {
      // one user key is a prefix of the other: the comparison continues into the suffix bytes
      // of the shorter key (internal keys are compared as plain byte strings here,
      // block_builder.cc:363-365)
      uint8_t a[8], b[8];
      const uint64_t sa = kept_suffix(rec, d, S), sb = kept_suffix(prec, pd, S);
      for (int q = 0; q < 8; q++) { a[q] = static_cast<uint8_t>(sa >> (8 * q)); b[q] = static_cast<uint8_t>(sb >> (8 * q)); }
      const uint32_t minlen = min(klen, static_cast<uint32_t>(pd.klen));
      while (shared < minlen) {
        const uint8_t x = shared < ulen ? rec[shared] : a[shared - ulen];
        const uint8_t y = shared < pul ? prec[shared] : b[shared - pul];
        if (x != y) break;
        shared++;
      }
    }
  }
  uint32_t nr, rs;
  if (E.key_encoding == 2) {
    // three_shared_parts: restart entries carry (value_size << 2) and the key size, then the whole key
    const uint64_t v4 = static_cast<uint64_t>(vlen) << 2;
    rs = (v4 < (1ull << 28) ? varint_len(static_cast<uint32_t>(v4)) : 5u) + ((klen < 128) ? 1u : 1u + varint_len(klen)) + klen + vlen;
    nr = rs;
    if (j > 0) {
      const Desc pd = E.kept[j - 1];
      const uint8_t* prec = kept_rec(E, pd, S);
      const IKeyRef pk{prec, pd.klen - 8u, kept_suffix(prec, pd, S)}, kk{rec, ulen, kept_suffix(rec, d, S)};
      TspPlan pl;
      tsp_plan(pk, kk, vlen, false, shared, &pl);
      nr = pl.hdr_len + pl.ns1 + pl.ns2 + vlen;
    }
  } else {
    nr = varint_len(shared) + varint_len(klen - shared) + varint_len(vlen) + (klen - shared) + vlen;
    rs = 1 + varint_len(klen) + varint_len(vlen) + klen + vlen;
  }
  *nr_out = nr; *rs_out = rs; *shared_out = shared;
  return add;
}

// Bloom filter key length of a survivor (0 = none): the merge kernel's DocKey walk where it ran, the key record otherwise.
__device__ __forceinline__ uint32_t entry_fk_len(const EncView& E, int S, const Desc& d) {
  return E.fk_src ? E.fk_src[d.gid] : static_cast<uint32_t>(docdb_filter_prefix_len(kept_rec(E, d, S), static_cast<int>(d.klen - 8u)));
}

// ---- block planning, pass 1 of 3 ------------------------------------------------------------------------------------
// One read of every descriptor gives the per-entry arrays (nr, shared, D, fk_len, is_new) and, in the same pass, the
// chunk partials of the three scans that follow: sums of nr per SCAN_CHUNK entries (P), sums of D per residue class
// mod ri per QROWS rows of ri entries (QQ), counts of new filter keys per SCAN_CHUNK entries (filter-key ordinals).
// A CTA owns PLAN_CHUNK entries: two SCAN_CHUNKs, and QROWS rows at the largest restart interval (64), so every chunk
// of every scan lies inside one CTA and the partials need no zeroing and no global atomics.
//
// is_new marks the entries whose filter key is non-empty and differs from the last non-empty filter key before them
// ("no need to insert duplicate keys", block_based_table_builder.cc:514-528). Equal keys are adjacent, so the previous
// entry decides, through the shared-prefix length, unless entries without a filter key lie in between (walked over).
constexpr int SCAN_CHUNK = 4096;
constexpr int QROWS = 128;
constexpr int PLAN_CHUNK = 2 * SCAN_CHUNK;
constexpr int PLAN_QSLOTS = PLAN_CHUNK / QROWS;      // (QQ chunk, residue class) pairs per CTA, whatever ri is
__global__ void __launch_bounds__(256) k_plan_entries(EncView E, int S, uint8_t* is_new, unsigned long long* p_part, uint32_t pc,
                                                      unsigned long long* q_part /*[ri][qchunks]*/, uint32_t qchunks, uint32_t* k_part) {
  static_assert(PLAN_QSLOTS == 64 && SCAN_CHUNK % 256 == 0, "restart intervals up to 64 fit one CTA's slots");
  __shared__ unsigned long long s_p[2], s_q[PLAN_QSLOTS];
  __shared__ uint32_t s_k[2];
  if (threadIdx.x < 2) { s_p[threadIdx.x] = 0; s_k[threadIdx.x] = 0; }
  if (threadIdx.x < PLAN_QSLOTS) s_q[threadIdx.x] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const uint64_t base = static_cast<uint64_t>(blockIdx.x) * PLAN_CHUNK;
  const uint32_t col = threadIdx.x & (E.ri - 1);     // 256 and SCAN_CHUNK are multiples of ri: a thread stays in one residue class
  const uint32_t qshift = 7 + E.ri_shift;            // log2(QROWS * ri): entries per QQ chunk
  uint32_t my_add = 0;
  unsigned long long qacc = 0;                       // D of this thread's class in the QQ chunk `qcur`
  uint32_t qcur = 0;
  // the warp's 32 entries lie in one QQ chunk (>= 128 entries, aligned), so every lane flushes in the same round
  auto flush_q = [&]() {
    for (uint32_t o = 16; o >= E.ri && o; o >>= 1) qacc += __shfl_xor_sync(0xffffffffu, qacc, o);
    if (static_cast<uint32_t>(lane) < E.ri) atomicAdd(&s_q[(qcur << E.ri_shift) + col], qacc);
    qacc = 0;
  };
  for (int half = 0; half < 2; half++) {
    unsigned long long psum = 0;
    uint32_t ksum = 0;
    for (int r = 0; r < SCAN_CHUNK / 256; r++) {
      const uint32_t o = half * SCAN_CHUNK + r * 256 + threadIdx.x;
      const uint64_t j64 = base + o;
      const bool valid = j64 < E.n;
      const uint32_t j = static_cast<uint32_t>(j64);
      if ((o >> qshift) != qcur) { flush_q(); qcur = o >> qshift; }
      uint32_t fl = 0, shared = 0;
      Desc d{};
      if (valid) {
        d = E.kept[j];
        uint32_t nr, rs;
        my_add = max(my_add, entry_sizes(E, S, j, d, &nr, &rs, &shared));
        const int16_t D = static_cast<int16_t>(static_cast<int32_t>(rs) - static_cast<int32_t>(nr));
        E.nr[j] = nr; E.shared[j] = static_cast<uint16_t>(shared); E.D[j] = D;
        psum += nr;
        qacc += static_cast<unsigned long long>(static_cast<long long>(D));
        if (E.fk_len) { fl = entry_fk_len(E, S, d); E.fk_len[j] = static_cast<uint16_t>(fl); }
      }
      if (E.fk_len) {
        uint32_t pfl = __shfl_up_sync(0xffffffffu, fl, 1);
        if (valid) {
          uint8_t nw = 0;
          if (fl) {
            nw = 1;
            if (j > 0) {
              if (lane == 0) pfl = entry_fk_len(E, S, E.kept[j - 1]);
              if (pfl) nw = !(pfl == fl && shared >= fl);
              else {
                uint32_t i = j - 1;
                Desc pd = E.kept[i];
                while (i > 0 && !pfl) { i--; pd = E.kept[i]; pfl = entry_fk_len(E, S, pd); }
                if (pfl == fl) nw = common_prefix_len(kept_rec(E, d, S), fl, kept_rec(E, pd, S), fl) < fl;
              }
            }
          }
          is_new[j] = nw;
          ksum += nw;
        }
      }
    }
    for (int o = 16; o; o >>= 1) { psum += __shfl_xor_sync(0xffffffffu, psum, o); ksum += __shfl_xor_sync(0xffffffffu, ksum, o); }
    if (lane == 0) { atomicAdd(&s_p[half], psum); atomicAdd(&s_k[half], ksum); }
  }
  flush_q();
  // the most one entry can add to FlushBlockBySizePolicy's estimate (block_next skips ahead with it)
  my_add = __reduce_max_sync(0xffffffffu, my_add);
  if (lane == 0 && my_add) atomicMax(E.max_add, my_add);
  __syncthreads();
  if (threadIdx.x < 2) {
    const uint64_t chunk = static_cast<uint64_t>(blockIdx.x) * 2 + threadIdx.x;
    if (chunk < pc) { p_part[chunk] = s_p[threadIdx.x]; if (k_part) k_part[chunk] = s_k[threadIdx.x]; }
  }
  if (threadIdx.x < PLAN_QSLOTS) {
    const uint64_t qc = static_cast<uint64_t>(blockIdx.x) * (PLAN_QSLOTS >> E.ri_shift) + (threadIdx.x >> E.ri_shift);
    if (qc < qchunks) q_part[static_cast<size_t>(threadIdx.x & (E.ri - 1)) * qchunks + qc] = s_q[threadIdx.x];
  }
}

// ---- scans: P = exclusive prefix of nr (u64); QQ = per-residue-class inclusive prefix of D ------
// Exclusive scan of a u64 array in place with one CTA of 1024 threads (loops past 1024 elements).
__device__ __forceinline__ void scan_u64_cta(unsigned long long* a, uint32_t n, unsigned long long* total) {
  __shared__ unsigned long long ws[32];
  __shared__ unsigned long long carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (uint32_t base = 0; base < n; base += 1024) {
    uint32_t i = base + threadIdx.x;
    unsigned long long v = i < n ? a[i] : 0, x = v;
    for (int o = 1; o < 32; o <<= 1) { unsigned long long y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) ws[wid] = x;
    __syncthreads();
    if (wid == 0) {
      unsigned long long w = ws[lane];
      for (int o = 1; o < 32; o <<= 1) { unsigned long long y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
      ws[lane] = w;
    }
    __syncthreads();
    if (i < n) a[i] = carry + (wid ? ws[wid - 1] : 0) + x - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry += ws[31];
    __syncthreads();
  }
  if (threadIdx.x == 0 && total) *total = carry;
}
__global__ void __launch_bounds__(1024) k_scan_u64_single(unsigned long long* a, uint32_t n, unsigned long long* total) { scan_u64_cta(a, n, total); }
// Block planning, pass 2 of 3: the chunk partials of k_plan_entries, one CTA per array. CTA 0: nr sums, CTA 1: new filter
// key counts (their total is the number of distinct filter keys), CTA 2 + c: D sums of residue class c.
__global__ void __launch_bounds__(1024) k_plan_scan(unsigned long long* p_part, uint32_t pc, unsigned long long* q_part, uint32_t qchunks,
                                                    uint32_t* k_part, uint32_t* n_keys) {
  if (blockIdx.x == 0) scan_u64_cta(p_part, pc, nullptr);
  else if (blockIdx.x == 1) { if (k_part) scan_u32_cta(k_part, pc, n_keys); }
  else scan_u64_cta(q_part + static_cast<size_t>(blockIdx.x - 2) * qchunks, qchunks, nullptr);
}
// Exclusive scan of a long u64 array in place (block sizes -> file offsets): chunk sums, one-CTA scan of the chunk sums
// (k_scan_u64_single), then every chunk scans itself from its base.
__global__ void __launch_bounds__(256) k_u64_chunk_sums(const unsigned long long* a, uint32_t n, unsigned long long* partial) {
  __shared__ unsigned long long sh;
  if (threadIdx.x == 0) sh = 0;
  __syncthreads();
  unsigned long long s = 0;
  const uint64_t base = static_cast<uint64_t>(blockIdx.x) * SCAN_CHUNK;
  for (uint32_t j = threadIdx.x; j < SCAN_CHUNK; j += 256) { const uint64_t i = base + j; if (i < n) s += a[i]; }
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(&sh, s);
  __syncthreads();
  if (threadIdx.x == 0) partial[blockIdx.x] = sh;
}
__global__ void __launch_bounds__(256) k_u64_chunk_final(unsigned long long* a, uint32_t n, const unsigned long long* partial) {
  __shared__ unsigned long long ws[8];
  const uint64_t base = static_cast<uint64_t>(blockIdx.x) * SCAN_CHUNK;
  constexpr int PER = SCAN_CHUNK / 256;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned long long v[PER], s = 0;
  for (int j = 0; j < PER; j++) { const uint64_t i = base + threadIdx.x * PER + j; v[j] = i < n ? a[i] : 0; s += v[j]; }
  unsigned long long x = s;
  for (int o = 1; o < 32; o <<= 1) { const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  if (lane == 31) ws[wid] = x;
  __syncthreads();
  unsigned long long run = partial[blockIdx.x] + x - s;
  for (int w = 0; w < wid; w++) run += ws[w];
  for (int j = 0; j < PER; j++) {
    const uint64_t i = base + threadIdx.x * PER + j;
    if (i < n) a[i] = run;
    run += v[j];
  }
}
// Block planning, pass 3 of 3. CTAs below pc take one SCAN_CHUNK each, a warp per 512 consecutive entries, 32 at a time
// (coalesced): P from nr and, with a filter policy, the survivor that introduces filter key `ord` (new_entry[ord]) and
// that key's bloom hash (hashes[ord]: the merge kernel's where it computed one, the key record's otherwise; nullptr
// when the filter blocks are built from the records). The CTAs above them write QQ: rows of ri entries, thread =
// (chunk of QROWS rows, residue class).
__global__ void __launch_bounds__(256) k_plan_final(EncView E, int S, const uint8_t* is_new, const unsigned long long* p_part, uint32_t pc,
                                                    const unsigned long long* q_part, uint32_t qchunks, const uint32_t* k_part,
                                                    uint32_t* new_entry, uint32_t* hashes) {
  if (blockIdx.x >= pc) {
    const uint32_t t = (blockIdx.x - pc) * blockDim.x + threadIdx.x;
    const uint32_t chunk = t >> E.ri_shift, col = t & (E.ri - 1);
    if (chunk >= qchunks) return;
    unsigned long long s = q_part[static_cast<size_t>(col) * qchunks + chunk];
    for (int r = 0; r < QROWS; r++) {
      const uint64_t i = ((static_cast<uint64_t>(chunk) * QROWS + r) << E.ri_shift) + col;
      if (i < E.n) { s += static_cast<unsigned long long>(static_cast<long long>(E.D[i])); E.QQ[i] = s; }
    }
    return;
  }
  constexpr int NW = 256 / 32, PER_WARP = SCAN_CHUNK / NW;
  __shared__ unsigned long long w_p[NW];
  __shared__ uint32_t w_k[NW];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint64_t wbase = static_cast<uint64_t>(blockIdx.x) * SCAN_CHUNK + static_cast<uint64_t>(wid) * PER_WARP;
  unsigned long long ps = 0;
  uint32_t ks = 0;
  for (int r = 0; r < PER_WARP; r += 32) {
    const uint64_t i = wbase + r + lane;
    if (i < E.n) { ps += E.nr[i]; if (is_new) ks += is_new[i]; }
  }
  for (int o = 16; o; o >>= 1) { ps += __shfl_xor_sync(0xffffffffu, ps, o); ks += __shfl_xor_sync(0xffffffffu, ks, o); }
  if (lane == 0) { w_p[wid] = ps; w_k[wid] = ks; }
  __syncthreads();
  unsigned long long run = p_part[blockIdx.x];
  uint32_t ord = is_new ? k_part[blockIdx.x] : 0;
  for (int w = 0; w < wid; w++) { run += w_p[w]; ord += w_k[w]; }
  for (int r = 0; r < PER_WARP; r += 32) {
    const uint64_t i = wbase + r + lane;
    const unsigned long long v = i < E.n ? E.nr[i] : 0;
    unsigned long long x = v;
    for (int o = 1; o < 32; o <<= 1) { const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (i < E.n) E.P[i] = run + x - v;
    if (i + 1 == E.n) E.P[E.n] = run + x;
    run += __shfl_sync(0xffffffffu, x, 31);
    if (is_new) {
      const bool nw = i < E.n && is_new[i];
      const uint32_t m = __ballot_sync(0xffffffffu, nw);
      if (nw) {
        const uint32_t o = ord + __popc(m & ((1u << lane) - 1));
        new_entry[o] = static_cast<uint32_t>(i);
        if (hashes) {
          const Desc d = E.kept[i];
          hashes[o] = E.fkh_src ? E.fkh_src[d.gid] : leveldb_hash(kept_rec(E, d, S), E.fk_len[i], kBloomSeed);
        }
      }
      ord += __popc(m);
    }
  }
}

// BlockBuilder::CurrentSizeEstimate after entries s..j of a block that started at s.
__device__ __forceinline__ unsigned long long blk_cur(const EncView& E, uint32_t s, uint32_t j) {
  const uint32_t t = (j - s) >> E.ri_shift;
  return (E.P[j + 1] - E.P[s]) + (E.QQ[s + (t << E.ri_shift)] - E.QQ[s] + static_cast<unsigned long long>(static_cast<long long>(E.D[s]))) + 4ull * (t + 1) + 4ull;
}

// next[s]: first entry of the block after the one starting at s (flush_block_policy.cc:45-76).
// thresh = block_size * (100 - deviation) (the rule is cur * 100 > thresh), madd = *E.max_add.
__device__ __forceinline__ uint32_t block_next(const EncView& E, uint32_t s, unsigned long long thresh, unsigned long long madd) {
  const unsigned long long BS = E.block_size;
  {
    // smallest m in (s, n] such that the block [s, m) satisfies cur*100 > thresh (or m == n)
    uint32_t lo = s + 1, hi = E.n;
    if (E.deviation == 0) {
      // only rule 1 (cur >= BS)
      while (lo < hi) { uint32_t mid = lo + ((hi - lo) >> 1); if (blk_cur(E, s, mid - 1) >= BS) hi = mid; else lo = mid + 1; }
      return lo;
    }
    // The second search below looks for the first m with cur(m - 1) > BS - madd. Where that bound is itself past the
    // deviation threshold, its answer cannot lie before the first search's (cur is monotone), so the first search is
    // skipped: half the probes.
    const bool second_only = BS > madd && (BS - madd) * 100 >= thresh;
    if (!second_only) {
      // interpolation: entries of one block have similar sizes, so "bytes still missing / bytes per entry so far" lands
      // within an entry or two of the answer; every probe tightens [lo, hi) (the predicate is monotone), the binary
      // search below finishes whatever is left (a probe costs two or three L2 round trips — this is what the kernel
      // is made of: ~4 probes per start instead of ~10 with galloping + bisection)
      uint32_t m = s + E.guess + (E.guess >> 3);
      for (int it = 0; it < 3 && lo < hi; it++) {
        if (m < lo) m = lo;
        if (m > hi) m = hi;
        const unsigned long long cur = blk_cur(E, s, m - 1);
        const unsigned long long have = cur * 100;
        const unsigned long long bpe = cur / (m - s) + 1;                      // bytes per entry so far (>= 1)
        if (have > thresh) {
          hi = m;
          const unsigned long long over = (have - thresh) / 100;
          const unsigned long long back = over / bpe + 1;
          m = back >= m - s ? s + 1 : m - static_cast<uint32_t>(back);
        } else {
          lo = m < E.n ? m + 1 : E.n;
          const unsigned long long miss = (thresh - have) / 100;
          const unsigned long long fwd = miss / bpe + 1;
          m = fwd >= E.n - m ? E.n : m + static_cast<uint32_t>(fwd);
        }
      }
      while (lo < hi) {
        uint32_t mid = lo + ((hi - lo) >> 1);
        if (blk_cur(E, s, mid - 1) * 100 > thresh) hi = mid; else lo = mid + 1;
      }
    }
    uint32_t m = lo;
    if (m < E.n && BS > madd) {
      // The scan below ends at the first m with cur(m - 1) >= BS or cur(m - 1) + add(m) > BS; no entry adds more than
      // `madd`, so every m with cur(m - 1) <= BS - madd can be skipped — cur is monotone: interpolate to that point
      // (the walk from 90 % to 100 % of a block is ~10 entries, each a round of dependent loads).
      const unsigned long long lim = BS - madd;
      uint32_t a = m, b = E.n, g = second_only ? s + E.guess + (E.guess >> 3) : m;
      for (int it = 0; it < 3 && a < b; it++) {
        if (g < a) g = a;
        if (g > b) g = b;
        const unsigned long long c = blk_cur(E, s, g - 1);
        const unsigned long long bpe = c / (g - s) + 1;
        if (c > lim) {
          b = g;
          const unsigned long long back = (c - lim) / bpe + 1;
          g = back >= g - a ? a : g - static_cast<uint32_t>(back);
        } else {
          a = g < E.n ? g + 1 : E.n;
          const unsigned long long fwd = (lim - c) / bpe + 1;
          g = fwd >= E.n - g ? E.n : g + static_cast<uint32_t>(fwd);
        }
      }
      while (a < b) {
        const uint32_t mid = a + ((b - a) >> 1);
        if (blk_cur(E, s, mid - 1) > lim) b = mid; else a = mid + 1;
      }
      m = a;
    }
    while (m < E.n) {
      const unsigned long long cur = blk_cur(E, s, m - 1);
      if (cur >= BS) break;
      const Desc d = E.kept[m];
      const unsigned long long est = cur + d.klen + d.vlen_out + ((((m - s) & (E.ri - 1)) == 0) ? 4 : 0) + 4 +
                                     varint_len(d.klen) + varint_len(d.vlen_out);
      if (est > BS && cur * 100 > thresh) break;
      m++;
    }
    return m;
  }
}

// next[s] for every entry of a segment, then exit1[s] = first chain element at or beyond the end of s's segment. One
// CTA per segment: next[] goes straight into the shared array the pointer jumping runs over (every update replaces a
// chain element by a later element of the same chain, so unsynchronised reads of neighbours are harmless).
__global__ void __launch_bounds__(256, 6) k_seg_exit(EncView E) {
  __shared__ uint32_t ex[SEG];
  const uint64_t b = static_cast<uint64_t>(blockIdx.x) * SEG;
  if (b >= E.n) return;
  const uint32_t e = static_cast<uint32_t>(umin64(b + SEG, E.n));
  const uint32_t cnt = e - static_cast<uint32_t>(b);
  const unsigned long long thresh = static_cast<unsigned long long>(E.block_size) * (100 - E.deviation), madd = *E.max_add;
  for (uint32_t i = threadIdx.x; i < cnt; i += blockDim.x) {
    const uint32_t m = block_next(E, static_cast<uint32_t>(b) + i, thresh, madd);
    ex[i] = m;
    E.next[b + i] = m;
  }
  __syncthreads();
  for (;;) {
    int changed = 0;
    for (uint32_t i = threadIdx.x; i < cnt; i += blockDim.x) {
      const uint32_t v = reinterpret_cast<volatile uint32_t*>(ex)[i];
      if (v < e) { reinterpret_cast<volatile uint32_t*>(ex)[i] = reinterpret_cast<volatile uint32_t*>(ex)[v - static_cast<uint32_t>(b)]; changed = 1; }
    }
    if (!__syncthreads_or(changed)) break;
  }
  for (uint32_t i = threadIdx.x; i < cnt; i += blockDim.x) E.exit1[b + i] = ex[i];
}

// gexit[g][q]: for a chain element at offset q inside the FIRST segment of group g, the first
// chain element at or beyond the end of the group.
__global__ void __launch_bounds__(256) k_group_exit(EncView E, uint32_t* gexit, uint32_t ngroups) {
  const uint64_t t = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x;
  const uint32_t g = static_cast<uint32_t>(t / SEG), q = static_cast<uint32_t>(t % SEG);
  if (g >= ngroups) return;
  const uint64_t gb = static_cast<uint64_t>(g) * SEG * GROUP_SEGS;
  const uint64_t ge = umin64(gb + static_cast<uint64_t>(SEG) * GROUP_SEGS, E.n);
  uint64_t s = gb + q;
  if (s >= E.n) { gexit[t] = E.n; return; }
  while (s < ge) s = E.exit1[s];
  gexit[t] = static_cast<uint32_t>(s);
}

// Serial walk over groups (one thread): group_first[g] = first chain element inside group g or
// 0xffffffff.
__global__ void k_chain_groups(EncView E, const uint32_t* gexit, uint32_t ngroups, uint32_t* group_first) {
  if (threadIdx.x || blockIdx.x) return;
  for (uint32_t g = 0; g < ngroups; g++) group_first[g] = 0xffffffffu;
  uint64_t s = 0;
  const uint64_t GS = static_cast<uint64_t>(SEG) * GROUP_SEGS;
  while (s < E.n) {
    const uint32_t g = static_cast<uint32_t>(s / GS);
    if (group_first[g] == 0xffffffffu) group_first[g] = static_cast<uint32_t>(s);
    const uint64_t q = s - g * GS;
    if (q < SEG) s = gexit[static_cast<uint64_t>(g) * SEG + q];
    else s = E.exit1[s];          // a block longer than a segment straddled the group boundary
  }
}

// Per group: walk segment exits from the group's first chain element, recording each segment's
// first chain element.
__global__ void __launch_bounds__(128) k_group_fill(EncView E, const uint32_t* group_first, uint32_t ngroups, uint32_t* seg_first, uint32_t nsegs) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= ngroups) return;
  const uint32_t s0 = static_cast<uint32_t>(g) * GROUP_SEGS, s1 = min(s0 + GROUP_SEGS, nsegs);
  for (uint32_t q = s0; q < s1; q++) seg_first[q] = 0xffffffffu;
  uint64_t s = group_first[g];
  if (s == 0xffffffffu) return;
  const uint64_t ge = umin64((static_cast<uint64_t>(g) + 1) * SEG * GROUP_SEGS, E.n);
  while (s < ge) {
    const uint32_t seg = static_cast<uint32_t>(s / SEG);
    if (seg_first[seg] == 0xffffffffu) seg_first[seg] = static_cast<uint32_t>(s);
    s = E.exit1[s];
  }
}

// Per segment: follow next[] from the segment's first chain element and count the blocks that start in it.
__global__ void __launch_bounds__(128) k_count_starts(EncView E, const uint32_t* seg_first, uint32_t nsegs, uint32_t* seg_blocks) {
  const uint32_t seg = blockIdx.x * blockDim.x + threadIdx.x;
  if (seg >= nsegs) return;
  uint64_t s = seg_first[seg];
  const uint64_t e = umin64((static_cast<uint64_t>(seg) + 1) * SEG, E.n);
  uint32_t c = 0;
  if (s != 0xffffffffu) while (s < e) { c++; s = E.next[s]; }
  seg_blocks[seg] = c;
}

// The same walk with seg_base = exclusive scan of those counts: block b starts at block_first[b]; block_off[b] = its size
// (contents incl. restart array + trailer, later scanned into file offsets); *max_size = the largest.
__global__ void __launch_bounds__(128) k_block_fill(EncView E, const uint32_t* seg_first, uint32_t nsegs, const uint32_t* seg_base,
                                                    uint32_t* block_first, unsigned long long* block_off, unsigned long long* max_size) {
  const uint32_t seg = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long mx = 0;
  if (seg < nsegs && seg_first[seg] != 0xffffffffu) {
    uint64_t s = seg_first[seg];
    const uint64_t e = umin64((static_cast<uint64_t>(seg) + 1) * SEG, E.n);
    uint32_t b = seg_base[seg];
    while (s < e) {
      const uint32_t nx = E.next[s];
      const unsigned long long sz = blk_cur(E, static_cast<uint32_t>(s), nx - 1) + 5;
      block_first[b] = static_cast<uint32_t>(s);
      block_off[b] = sz;
      mx = sz > mx ? sz : mx;
      b++;
      s = nx;
    }
  }
  for (int o = 16; o; o >>= 1) { const unsigned long long y = __shfl_xor_sync(0xffffffffu, mx, o); mx = y > mx ? y : mx; }
  if ((threadIdx.x & 31) == 0 && mx) atomicMax(max_size, mx);
}

__device__ __forceinline__ int put_varint(uint8_t* p, uint32_t v) {
  int n = 0;
  while (v >= 128) { p[n++] = static_cast<uint8_t>(v | 128); v >>= 7; }
  p[n++] = static_cast<uint8_t>(v);
  return n;
}

// ---- CRC32C -------------------------------------------------------------------------------------
// Reflected polynomial 0x82F63B78 (rocksdb/util/crc32c.cc). Each lane runs slicing-by-4 over its
// word range of the block, the 32 partial CRCs are combined with
//   crc(A || B) = x^(8|B|) * crc(A) + crc(B)   (mod P, reflected; zlib's crc32_combine identity).
__device__ uint32_t g_crc_tab[4][256];
__device__ uint32_t g_crc_x2n[32];      // x^(2^k) mod P
constexpr uint32_t CRC_XPOW_TABLE = 1u << 16;
__device__ uint32_t g_crc_xpow8[CRC_XPOW_TABLE + 1];   // x^(8m) mod P for m = 0..65536 bytes
// Strided CRC (k_encode_smem): multiplying the register by x^(8 * 1024) (256 words further from the
// end of the message) is a fixed GF(2)-linear map and so costs the same four lookups as the
// ordinary one-word step; g_crc_stride[3 - b][x] = (x << 8b) * x^(8 * 1024) mod P.
constexpr uint32_t CRC_STRIDE_WORDS = 256;
__device__ uint32_t g_crc_stride[4][256];
__device__ uint32_t g_crc_s32[4][256];                 // the same for a stride of 32 words (one warp): (x << 8b) * x^(8 * 128) mod P

__global__ void k_crc_init() {
  const uint32_t i = threadIdx.x;
  uint32_t c = i;
  for (int k = 0; k < 8; k++) c = (c >> 1) ^ ((c & 1) ? 0x82F63B78u : 0u);
  g_crc_tab[0][i] = c;
  __syncthreads();
  for (int t = 1; t < 4; t++) {
    uint32_t prev = g_crc_tab[t - 1][i];
    g_crc_tab[t][i] = (prev >> 8) ^ g_crc_tab[0][prev & 0xff];
    __syncthreads();
  }
  if (i == 0) {
    auto mul = [](uint32_t a, uint32_t b) {
      uint32_t m = 1u << 31, p = 0;
      for (;;) {
        if (a & m) { p ^= b; if ((a & (m - 1)) == 0) break; }
        m >>= 1;
        b = (b & 1) ? (b >> 1) ^ 0x82F63B78u : b >> 1;
      }
      return p;
    };
    uint32_t p = 1u << 30;                      // x^1
    g_crc_x2n[0] = p;
    for (int n = 1; n < 32; n++) { p = mul(p, p); g_crc_x2n[n] = p; }
  }
}

__device__ __forceinline__ uint32_t crc_mulmod(uint32_t a, uint32_t b) {
  uint32_t m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) { p ^= b; if ((a & (m - 1)) == 0) break; }
    m >>= 1;
    b = (b & 1) ? (b >> 1) ^ 0x82F63B78u : b >> 1;
  }
  return p;
}
// The same product without the bit-serial loop. In the reflected representation (bit 31 = x^0) the carry-less
// product of two registers, shifted left by one, holds the 63-coefficient product with x^0..x^31 in its HIGH word
// and x^32..x^62 in its LOW word; (low word) * x^32 mod P is the ordinary four-byte zero step of the CRC, so
//   a * b mod P = step32(lo(z << 1)) ^ hi(z << 1),   z = clmul(a, b).
// The carry-less multiplication itself uses integer multipliers: with the operands split into four classes of bit
// positions (mod 4), every product bit sums at most eight partial products — the carries stay inside the 4-bit
// group and the group's lowest bit is the XOR. Reduction is linear: products are XOR-accumulated unreduced
// (crc_clmul) and reduced once (crc_clmul_reduce).
__device__ __forceinline__ unsigned long long crc_clmul(uint32_t x, uint32_t y) {
  const uint32_t x0 = x & 0x11111111u, x1 = x & 0x22222222u, x2 = x & 0x44444444u, x3 = x & 0x88888888u;
  const uint32_t y0 = y & 0x11111111u, y1 = y & 0x22222222u, y2 = y & 0x44444444u, y3 = y & 0x88888888u;
#define YB_M64(a, b) (static_cast<unsigned long long>(a) * (b))
  const unsigned long long z0 = YB_M64(x0, y0) ^ YB_M64(x1, y3) ^ YB_M64(x2, y2) ^ YB_M64(x3, y1);
  const unsigned long long z1 = YB_M64(x0, y1) ^ YB_M64(x1, y0) ^ YB_M64(x2, y3) ^ YB_M64(x3, y2);
  const unsigned long long z2 = YB_M64(x0, y2) ^ YB_M64(x1, y1) ^ YB_M64(x2, y0) ^ YB_M64(x3, y3);
  const unsigned long long z3 = YB_M64(x0, y3) ^ YB_M64(x1, y2) ^ YB_M64(x2, y1) ^ YB_M64(x3, y0);
#undef YB_M64
  return (z0 & 0x1111111111111111ull) | (z1 & 0x2222222222222222ull) | (z2 & 0x4444444444444444ull) | (z3 & 0x8888888888888888ull);
}
// tab(b) = g_crc_tab[0][b] from wherever the caller keeps the byte table
template <class Tab>
__device__ __forceinline__ uint32_t crc_clmul_reduce(unsigned long long z, Tab tab) {
  z <<= 1;
  uint32_t c = static_cast<uint32_t>(z);
#pragma unroll
  for (int i = 0; i < 4; i++) c = tab(c & 0xff) ^ (c >> 8);
  return c ^ static_cast<uint32_t>(z >> 32);
}
// x^(8 * nbytes) mod P
__device__ __forceinline__ uint32_t crc_xpow_bytes(uint64_t nbytes, const uint32_t* x2n) {
  uint32_t p = 1u << 31;                         // x^0
  uint32_t k = 3;
  while (nbytes) {
    if (nbytes & 1) p = crc_mulmod(x2n[k & 31], p);
    nbytes >>= 1; k++;
  }
  return p;
}

__global__ void k_crc_init_xpow() {
  const uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m <= CRC_XPOW_TABLE) g_crc_xpow8[m] = crc_xpow_bytes(m, g_crc_x2n);
  if (m < 1024) {
    const uint32_t xp = crc_xpow_bytes(4 * CRC_STRIDE_WORDS, g_crc_x2n);
    const uint32_t r = m >> 8, x = m & 255;
    g_crc_stride[r][x] = crc_mulmod(xp, x << (8 * (3 - r)));
  }
  if (m < 1024) {
    const uint32_t xp = crc_xpow_bytes(4 * 32, g_crc_x2n);
    const uint32_t r = m >> 8, x = m & 255;
    g_crc_s32[r][x] = crc_mulmod(xp, x << (8 * (3 - r)));
  }
}
// crc * x^(8 nbytes): table lookup + one modular multiplication for the common distances.
__device__ __forceinline__ uint32_t crc_shift(uint32_t crc, uint64_t nbytes, const uint32_t* x2n) {
  if (nbytes == 0) return crc;
  const uint32_t m = nbytes <= CRC_XPOW_TABLE ? __ldg(&g_crc_xpow8[nbytes]) : crc_xpow_bytes(nbytes, x2n);
  return crc_mulmod(m, crc);
}

// CRC32C of [p, p+len) computed by one warp. Returns the finalized CRC in every lane.
__device__ uint32_t warp_crc32c(const uint8_t* p, uint64_t len, int lane, const uint32_t (*tab)[256], const uint32_t* x2n) {
  // head bytes up to 4-byte alignment, body words split evenly over lanes, tail bytes
  uint32_t head = static_cast<uint32_t>((4 - (reinterpret_cast<uintptr_t>(p) & 3)) & 3);
  if (head > len) head = static_cast<uint32_t>(len);
  const uint64_t nwords = (len - head) >> 2;
  const uint32_t tail = static_cast<uint32_t>((len - head) & 3);
  const uint32_t* w = reinterpret_cast<const uint32_t*>(p + head);
  const uint64_t per = (nwords + 31) / 32;
  const uint64_t w0 = umin64(per * lane, nwords), w1 = umin64(w0 + per, nwords);
  uint32_t acc = 0;
  if (w1 > w0) {
    uint32_t c = 0xffffffffu;
    for (uint64_t i = w0; i < w1; i++) {
      c ^= w[i];
      c = tab[3][c & 0xff] ^ tab[2][(c >> 8) & 0xff] ^ tab[1][(c >> 16) & 0xff] ^ tab[0][c >> 24];
    }
    c = ~c;
    const uint64_t after = (nwords - w1) * 4 + tail;
    acc = crc_shift(c, after, x2n);
  }
  if (lane == 0 && head) {
    uint32_t c = 0xffffffffu;
    for (uint32_t i = 0; i < head; i++) c = tab[0][(c ^ p[i]) & 0xff] ^ (c >> 8);
    c = ~c;
    const uint64_t after = len - head;
    acc ^= crc_shift(c, after, x2n);
  }
  if (lane == 31 && tail) {
    uint32_t c = 0xffffffffu;
    const uint8_t* q = p + len - tail;
    for (uint32_t i = 0; i < tail; i++) c = tab[0][(c ^ q[i]) & 0xff] ^ (c >> 8);
    acc ^= ~c;
  }
  for (int o = 16; o; o >>= 1) acc ^= __shfl_xor_sync(0xffffffffu, acc, o);
  return acc;
}

__device__ __forceinline__ uint32_t crc_mask(uint32_t c) { return ((c >> 15) | (c << 17)) + 0xa282ead8u; }

// CRC32C of [p, p+len) in global memory by one warp with COALESCED reads: the words are numbered from
// the end, lane l folds the words at distance l, l+32, ... with the map "multiply by x^(8*128)"
// (s32, four lookups per word like an ordinary step), then multiplies its partial by x^(32(l+1)) (kc)
// and the lanes XOR. Leading bytes up to word alignment seed the register (folded into word 0),
// trailing bytes are stepped at the end. Returns the finalized CRC in every lane.
__device__ uint32_t warp_crc32c_strided(const uint8_t* p, uint64_t len, int lane, const uint32_t* tab0, const uint32_t (*s32)[256], uint32_t kc) {
  uint32_t head = static_cast<uint32_t>((4 - (reinterpret_cast<uintptr_t>(p) & 3)) & 3);
  if (head > len) head = static_cast<uint32_t>(len);
  uint32_t c1 = 0xffffffffu;
  for (uint32_t i = 0; i < head; i++) c1 = tab0[(c1 ^ p[i]) & 0xff] ^ (c1 >> 8);
  const uint64_t nwords = (len - head) >> 2;
  const uint32_t tail = static_cast<uint32_t>((len - head) & 3);
  const uint32_t* w = reinterpret_cast<const uint32_t*>(p + head);
  uint32_t acc = 0;
  if (nwords > static_cast<uint64_t>(lane)) {
    const uint64_t last = nwords - 1 - lane;
    uint64_t i = last & 31;
    acc = __ldg(w + i);
    if (i == 0) acc ^= c1;
    i += 32;
    // eight independent loads in flight per lane, then the dependent fold
    for (; i + 7 * 32 <= last; i += 8 * 32) {
      uint32_t nx[8];
#pragma unroll
      for (int u = 0; u < 8; u++) nx[u] = __ldg(w + i + 32 * u);
#pragma unroll
      for (int u = 0; u < 8; u++) {
        acc = s32[3][acc & 0xff] ^ s32[2][(acc >> 8) & 0xff] ^ s32[1][(acc >> 16) & 0xff] ^ s32[0][acc >> 24];
        acc ^= nx[u];
      }
    }
    for (; i <= last; i += 32) {
      const uint32_t nx = __ldg(w + i);
      acc = s32[3][acc & 0xff] ^ s32[2][(acc >> 8) & 0xff] ^ s32[1][(acc >> 16) & 0xff] ^ s32[0][acc >> 24];
      acc ^= nx;
    }
  }
  uint32_t r = acc ? crc_mulmod(kc, acc) : 0u;
  for (int o = 16; o; o >>= 1) r ^= __shfl_xor_sync(0xffffffffu, r, o);
  if (nwords == 0) r = c1;
  const uint8_t* q = p + len - tail;
  for (uint32_t i = 0; i < tail; i++) r = tab0[(r ^ q[i]) & 0xff] ^ (r >> 8);
  return ~r;
}

// mode 0: write trailers of freshly encoded blocks. mode 1: verify stored trailers (inputs). mode 2: verify the stored
// trailers of a finished table for the output check, which reports the lowest failing block (JobDev::verify_fail).
__global__ void __launch_bounds__(256) k_crc_blocks(uint8_t* file, const unsigned long long* off, const uint32_t* size32,
                                                    const unsigned long long* size_from_next, uint32_t nblocks, int mode, JobDev* J) {
  __shared__ uint32_t tab0[256];
  __shared__ uint32_t s32[4][256];
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) (&s32[0][0])[i] = (&g_crc_s32[0][0])[i];
  tab0[threadIdx.x] = g_crc_tab[0][threadIdx.x];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const uint32_t kc = g_crc_xpow8[4 * (lane + 1)];                 // x^(32 (lane + 1))
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t b = warp; b < nblocks; b += nwarps) {
    const unsigned long long o = off[b];
    // contents length (without the 5-byte trailer)
    const uint64_t len = size32 ? size32[b] : (size_from_next[b + 1] - o - 5);
    uint8_t* p = file + o;
    const uint32_t crc = crc_mask(warp_crc32c_strided(p, len + 1, lane, tab0, s32, kc));   // block + type byte
    if (mode == 0) {
      if (lane < 4) p[len + 1 + lane] = static_cast<uint8_t>(crc >> (8 * lane));
    } else {
      const uint32_t stored = ldg_u32_unaligned(p + len + 1);
      if (lane == 0 && stored != crc) {
        if (mode == 2) atomicMin(&J->verify_fail, verify_pack(b, 0, VERIFY_CHECKSUM));
        else dev_fail(J, DEV_ERR_BAD_CRC, b);
      }
    }
  }
}

// Bytes [sh, sh + 16) of the 32-byte pair (a, b).
__device__ __forceinline__ uint4 shift16(const uint4& a, const uint4& b, uint32_t sh) {
  uint32_t w0 = a.x, w1 = a.y, w2 = a.z, w3 = a.w, w4 = b.x, w5 = b.y, w6 = b.z, w7 = b.w;
  const uint32_t q = sh >> 2, bits = (sh & 3) * 8;
  if (q & 1) { w0 = w1; w1 = w2; w2 = w3; w3 = w4; w4 = w5; w5 = w6; w6 = w7; }
  if (q & 2) { w0 = w2; w1 = w3; w2 = w4; w3 = w5; w4 = w6; }
  uint4 o;
  o.x = __funnelshift_r(w0, w1, bits); o.y = __funnelshift_r(w1, w2, bits);
  o.z = __funnelshift_r(w2, w3, bits); o.w = __funnelshift_r(w3, w4, bits);
  return o;
}

// Bytes [from, to) of a 16-byte-aligned record in global memory into shared memory (any
// alignment): the record is fetched as 16-byte vectors (all in flight together), the 4-byte
// shared stores are funnel-shifted out of registers; single bytes only at the two ends.
// Reads record bytes up to ((to + 3) & ~3) + 4 at most (inside the record stride).
__device__ __forceinline__ void copy_rec_to_smem(uint8_t* dst, const uint8_t* rec, uint32_t from, uint32_t to) {
  uint32_t n = to - from;
  while (n && (reinterpret_cast<uintptr_t>(dst) & 3)) { *dst++ = __ldg(rec + from); from++; n--; }
  const uint32_t nw = n >> 2;
  if (nw) {
    const uint32_t w1 = from >> 2, bits = (from & 3) * 8;
    const uint32_t wend = w1 + nw + (bits ? 1 : 0);            // source words [w1, wend)
    uint32_t* dw = reinterpret_cast<uint32_t*>(dst);
    const uint4* rv = reinterpret_cast<const uint4*>(rec);
    uint32_t prev = 0;
    for (uint32_t c = w1 >> 2; c * 4 < wend; c++) {
      const uint4 v = __ldg(rv + c);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int t = 0; t < 4; t++) {
        const uint32_t j = c * 4 + t;
        if (bits) { if (j > w1 && j - 1 - w1 < nw) dw[j - 1 - w1] = __funnelshift_r(prev, w[t], bits); }
        else if (j >= w1 && j - w1 < nw) dw[j - w1] = w[t];
        prev = w[t];
      }
    }
  }
  for (uint32_t i = nw * 4; i < n; i++) dst[i] = __ldg(rec + from + i);
}

// Internal-key bytes [from, to) of a survivor (user key from the record, then the 8-byte suffix).
__device__ __forceinline__ uint8_t* copy_ikey(uint8_t* p, const uint8_t* rec, uint32_t ulen, uint64_t suffix, uint32_t from, uint32_t to) {
  if (from < ulen && from < to) {
    const uint32_t e = to < ulen ? to : ulen;
    copy_rec_to_smem(p, rec, from, e);
    p += e - from; from = e;
  }
  for (uint32_t i = from; i < to; i++) *p++ = static_cast<uint8_t>(suffix >> (8 * (i - ulen)));
  return p;
}

// Entry header + key delta of survivor j at p, either key encoding (BlockBuilder::Add,
// table/block_builder.cc:347-412). Returns the position of the value.
template <int ENC>
__device__ __forceinline__ uint8_t* emit_entry_key(const EncView& E, int S, uint32_t j, const Desc& d, const uint8_t* rec, uint64_t suffix,
                                                   bool restart, uint8_t* p) {
  const uint32_t klen = d.klen, ulen = klen - 8u, vlen = d.vlen_out;
  if (ENC != 2) {
    const uint32_t shared = restart ? 0u : E.shared[j];
    p += put_varint(p, shared);
    p += put_varint(p, klen - shared);
    p += put_varint(p, vlen);
    return copy_ikey(p, rec, ulen, suffix, shared, klen);
  }
  TspPlan pl;
  const IKeyRef kk{rec, ulen, suffix};
  if (restart) {
    const IKeyRef none{nullptr, 0, 0};
    tsp_plan(none, kk, vlen, true, 0, &pl);
  } else {
    const Desc pd = E.kept[j - 1];
    const uint8_t* prec = kept_rec(E, pd, S);
    const IKeyRef pk{prec, pd.klen - 8u, kept_suffix(prec, pd, S)};
    tsp_plan(pk, kk, vlen, false, E.shared[j], &pl);
  }
  for (uint32_t i = 0; i < pl.hdr_len; i++) *p++ = pl.hdr[i];
  p = copy_ikey(p, rec, ulen, suffix, pl.shared, pl.shared + pl.ns1);
  const uint32_t b2 = klen - pl.last_reuse - pl.ns2;
  return copy_ikey(p, rec, ulen, suffix, b2, b2 + pl.ns2);
}

// ---- fused encoder (v2): one CTA per output block -------------------------------------------
// Phase A  one thread per entry: header + key delta (few bytes) straight to HBM, value copy job
//          into a shared-memory table.
// Phase B  the value bytes (the bulk) are moved as 16-byte destination-aligned vector stores;
//          every thread takes (entry, 16-B chunk) items from a flat list, sources are read as two
//          aligned 16-B loads and funnel-shifted into place.
// Phase C  restart array, count, trailer type byte.
// Phase D  CRC32C of the block while it is still hot in L1/L2 (no second pass over HBM), trailer.
constexpr int ENC_THREADS = 256;
constexpr int ENC_EMAX = 512;      // entries per pass through the shared-memory table
constexpr int ENC_ITEMS = 4096;    // direct item->entry map size (64 KB of values per pass)
constexpr int ENC_EM_S = 256;          // entries per pass in k_encode_smem (= ENC_THREADS)
constexpr int ENC_ITEMS_SMEM = 1024;   // items (runs of up to 4 value chunks) per pass in k_encode_smem: a 36 KB image has < 850

// 16 bytes starting at an arbitrary address: two aligned 16-byte loads + funnel shift. Reads
// [src & ~15, (src & ~15) + 32).
__device__ __forceinline__ uint4 load_unaligned16(const uint8_t* src) {
  const uint32_t sh = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(src) & 15);
  const uint4* sa = reinterpret_cast<const uint4*>(src - sh);
  const uint4 a = __ldg(sa);
  if (sh == 0) return a;
  const uint4 b = __ldg(sa + 1);
  uint32_t w0 = a.x, w1 = a.y, w2 = a.z, w3 = a.w, w4 = b.x, w5 = b.y, w6 = b.z, w7 = b.w;
  const uint32_t q = sh >> 2, bits = (sh & 3) * 8;
  if (q & 1) { w0 = w1; w1 = w2; w2 = w3; w3 = w4; w4 = w5; w5 = w6; w6 = w7; }
  if (q & 2) { w0 = w2; w1 = w3; w2 = w4; w3 = w5; w4 = w6; }
  uint4 o;
  o.x = __funnelshift_r(w0, w1, bits); o.y = __funnelshift_r(w1, w2, bits);
  o.z = __funnelshift_r(w2, w3, bits); o.w = __funnelshift_r(w3, w4, bits);
  return o;
}

__device__ __forceinline__ void copy_chunk16(uint8_t* dst_chunk, const uint8_t* src) {
  // dst_chunk 16-byte aligned; src arbitrary. Reads [src & ~15, (src & ~15) + 32).
  const uint32_t sh = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(src) & 15);
  const uint4* sa = reinterpret_cast<const uint4*>(src - sh);
  const uint4 a = __ldg(sa);
  if (sh == 0) { *reinterpret_cast<uint4*>(dst_chunk) = a; return; }
  const uint4 b = __ldg(sa + 1);
  uint32_t w0 = a.x, w1 = a.y, w2 = a.z, w3 = a.w, w4 = b.x, w5 = b.y, w6 = b.z, w7 = b.w;
  const uint32_t q = sh >> 2, bits = (sh & 3) * 8;
  if (q & 1) { w0 = w1; w1 = w2; w2 = w3; w3 = w4; w4 = w5; w5 = w6; w6 = w7; }
  if (q & 2) { w0 = w2; w1 = w3; w2 = w4; w3 = w5; w4 = w6; }
  uint4 o;
  o.x = __funnelshift_r(w0, w1, bits); o.y = __funnelshift_r(w1, w2, bits);
  o.z = __funnelshift_r(w2, w3, bits); o.w = __funnelshift_r(w3, w4, bits);
  *reinterpret_cast<uint4*>(dst_chunk) = o;
}

template <int ENC>
__global__ void __launch_bounds__(ENC_THREADS, 2) k_encode_fused(EncView E, int S, const uint32_t* block_first, uint32_t nblocks,
                                                                const unsigned long long* block_off, uint8_t* out, unsigned long long min_total) {
  __shared__ uint32_t tab[4][256];
  __shared__ uint32_t x2n[32];
  __shared__ unsigned long long t_dst[ENC_EMAX];     // absolute destination address of the value
  __shared__ unsigned long long t_src[ENC_EMAX];     // source address of the value
  __shared__ uint32_t t_len[ENC_EMAX];               // bytes to copy (0 = value written in phase A)
  __shared__ uint32_t t_chunk[ENC_EMAX + 1];         // exclusive prefix of 16-B chunk counts
  __shared__ uint16_t t_item[ENC_ITEMS];             // chunk item -> entry (when the pass has <= ENC_ITEMS items)
  __shared__ uint32_t warp_sums[32];
  __shared__ uint32_t warp_crc[ENC_THREADS / 32];
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) (&tab[0][0])[i] = (&g_crc_tab[0][0])[i];
  if (threadIdx.x < 32) x2n[threadIdx.x] = g_crc_x2n[threadIdx.x];
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  constexpr int NW = ENC_THREADS / 32;

  for (uint32_t b = blockIdx.x; b < nblocks; b += gridDim.x) {
    const uint32_t s = block_first[b], e = (b + 1 < nblocks) ? block_first[b + 1] : E.n;
    const unsigned long long boff = block_off[b];
    if (block_off[b + 1] - boff <= min_total) continue;              // handled by k_encode_smem
    const unsigned long long blen = block_off[b + 1] - boff - 5;     // contents length
    uint8_t* blk = out + boff;
    const unsigned long long Ps = E.P[s];
    const unsigned long long Qs = E.QQ[s] - static_cast<unsigned long long>(static_cast<long long>(E.D[s]));
    const uint32_t tl = (e - 1 - s) >> E.ri_shift;
    const unsigned long long body = (E.P[e] - Ps) + (E.QQ[s + (tl << E.ri_shift)] - Qs);

    for (uint32_t p0 = s; p0 < e; p0 += ENC_EMAX) {
      const uint32_t pn = min(static_cast<uint32_t>(ENC_EMAX), e - p0);
      // ---- phase A
      for (uint32_t q = threadIdx.x; q < pn; q += blockDim.x) {
        const uint32_t j = p0 + q;
        const bool restart = ((j - s) & (E.ri - 1)) == 0;
        unsigned long long off = E.P[j] - Ps;
        if (j > s) { const uint32_t tp = (j - 1 - s) >> E.ri_shift; off += E.QQ[s + (tp << E.ri_shift)] - Qs; }
        const Desc d = E.kept[j];
        const uint8_t* rec = kept_rec(E, d, S);
        const uint32_t vlen = d.vlen_out;
        uint8_t* p = emit_entry_key<ENC>(E, S, j, d, rec, kept_suffix(rec, d, S), restart, blk + off);
        const RunView& run = E.runs[d.run];
        const uint8_t* vs = run.data + run.val_off[d.gid - run.gid_base];
        uint32_t copy_len = vlen;
        if (d.flags & ENT_VAL_TOMBSTONE) { p[0] = 'X'; copy_len = 0; }
        else if (d.flags & ENT_VAL_REENCODE) {
          const ValueRewrite& rw = E.rewrites[d.rewrite_slot];
          for (uint32_t i = 0; i < rw.prefix_len; i++) p[i] = rw.prefix[i];
          const uint32_t rest = vlen - rw.prefix_len;
          for (uint32_t i = 0; i < rest; i++) p[rw.prefix_len + i] = vs[rw.skip + i];
          copy_len = 0;
        }
        t_dst[q] = reinterpret_cast<unsigned long long>(p);
        t_src[q] = reinterpret_cast<unsigned long long>(vs);
        t_len[q] = copy_len;
        if (restart) {
          const uint32_t t = (j - s) >> E.ri_shift;
          uint8_t* r = blk + body + 4ull * t;
          const uint32_t o32 = static_cast<uint32_t>(off);
          r[0] = static_cast<uint8_t>(o32); r[1] = static_cast<uint8_t>(o32 >> 8); r[2] = static_cast<uint8_t>(o32 >> 16); r[3] = static_cast<uint8_t>(o32 >> 24);
        }
      }
      __syncthreads();
      // chunk counts -> exclusive prefix (pn <= ENC_EMAX = 2 * blockDim)
      uint32_t c0 = 0, c1 = 0;
      {
        const uint32_t q0 = threadIdx.x * 2, q1 = q0 + 1;
        if (q0 < pn && t_len[q0]) { const unsigned long long d0 = t_dst[q0]; c0 = static_cast<uint32_t>((((d0 + t_len[q0] + 15) & ~15ull) - (d0 & ~15ull)) >> 4); }
        if (q1 < pn && t_len[q1]) { const unsigned long long d0 = t_dst[q1]; c1 = static_cast<uint32_t>((((d0 + t_len[q1] + 15) & ~15ull) - (d0 & ~15ull)) >> 4); }
      }
      uint32_t total_chunks;
      const uint32_t base = block_exclusive_scan(c0 + c1, warp_sums, &total_chunks);
      {
        const uint32_t q0 = threadIdx.x * 2;
        if (q0 < ENC_EMAX) { t_chunk[q0] = base; if (q0 + 1 <= ENC_EMAX) t_chunk[q0 + 1] = base + c0; }
        if (threadIdx.x == blockDim.x - 1) t_chunk[ENC_EMAX] = base + c0 + c1;
      }
      __syncthreads();
      const bool direct = total_chunks <= ENC_ITEMS;
      if (direct) {
        const uint32_t q0 = threadIdx.x * 2;
        for (uint32_t q = q0; q < q0 + 2 && q < pn; q++)
          for (uint32_t it = t_chunk[q]; it < t_chunk[q + 1]; it++) t_item[it] = static_cast<uint16_t>(q);
        __syncthreads();
      }
      // ---- phase B
      for (uint32_t it = threadIdx.x; it < total_chunks; it += blockDim.x) {
        uint32_t q;
        if (direct) q = t_item[it];
        else {
          uint32_t lo = 0, hi = pn;                   // last q with t_chunk[q] <= it
          while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (t_chunk[mid] <= it) lo = mid; else hi = mid; }
          q = lo;
        }
        const unsigned long long d0 = t_dst[q], d1 = d0 + t_len[q];
        const unsigned long long A = (d0 & ~15ull) + 16ull * (it - t_chunk[q]);
        const uint8_t* src = reinterpret_cast<const uint8_t*>(t_src[q]) + static_cast<long long>(A - d0);
        if (A >= d0 && A + 16 <= d1) {
          copy_chunk16(reinterpret_cast<uint8_t*>(A), src);
        } else {
          const unsigned long long lo_a = A > d0 ? A : d0, hi_a = (A + 16 < d1) ? A + 16 : d1;
          for (unsigned long long a = lo_a; a < hi_a; a++) *reinterpret_cast<uint8_t*>(a) = src[a - A];
        }
      }
      __syncthreads();
    }
    // ---- phase C
    if (threadIdx.x == 0) {
      const uint32_t nres = tl + 1;
      uint8_t* q = blk + body + 4ull * nres;
      q[0] = static_cast<uint8_t>(nres); q[1] = static_cast<uint8_t>(nres >> 8); q[2] = static_cast<uint8_t>(nres >> 16); q[3] = static_cast<uint8_t>(nres >> 24);
      q[4] = 0;   // kNoCompression
    }
    __syncthreads();
    // ---- phase D: CRC over contents + type byte, split over the warps
    const unsigned long long L = blen + 1;
    const unsigned long long per = (L + NW - 1) / NW;
    const unsigned long long a0 = umin64(per * wid, L), a1 = umin64(a0 + per, L);
    uint32_t c = 0;
    if (a1 > a0) {
      c = warp_crc32c(blk + a0, a1 - a0, lane, tab, x2n);
      const unsigned long long after = L - a1;
      c = crc_shift(c, after, x2n);
    }
    if (lane == 0) warp_crc[wid] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t crc = 0;
      for (int w = 0; w < NW; w++) crc ^= warp_crc[w];
      crc = crc_mask(crc);
      uint8_t* t = blk + blen + 1;
      t[0] = static_cast<uint8_t>(crc); t[1] = static_cast<uint8_t>(crc >> 8); t[2] = static_cast<uint8_t>(crc >> 16); t[3] = static_cast<uint8_t>(crc >> 24);
    }
    __syncthreads();
  }
}

// ---- shared-memory block assembler (v3): the whole block image is built in shared memory --------
// All byte-granular scatter (headers, key deltas, value edges, restart array) lands in shared
// memory; HBM sees only 16-byte vector loads of the source values and 16-byte vector stores of
// the finished image; the CRC is computed from the shared-memory image. Blocks larger than
// ENC_SMEM_CAP are left to k_encode_fused (only_big = 1).
constexpr uint32_t ENC_SMEM_CAP = 36 * 1024;       // bytes of block image (contents + trailer) per CTA

struct EncBlkHdr { unsigned long long boff; uint32_t btot, s, e; };
struct EncBlkSums { unsigned long long Ps, Qs; uint32_t body, tl; };
__device__ __forceinline__ EncBlkHdr enc_load_hdr(const EncView& E, const uint32_t* block_first, const unsigned long long* block_off,
                                                  uint32_t b, uint32_t nblocks) {
  EncBlkHdr h;
  h.boff = block_off[b];
  const unsigned long long t = block_off[b + 1] - h.boff;
  h.btot = t > 0xffffffffull ? 0xffffffffu : static_cast<uint32_t>(t);
  h.s = block_first[b];
  h.e = (b + 1 < nblocks) ? block_first[b + 1] : E.n;
  return h;
}
__device__ __forceinline__ EncBlkSums enc_load_sums(const EncView& E, const EncBlkHdr& h) {
  EncBlkSums u;
  u.Ps = E.P[h.s];
  u.Qs = E.QQ[h.s] - static_cast<unsigned long long>(static_cast<long long>(E.D[h.s]));
  u.tl = (h.e - 1 - h.s) >> E.ri_shift;
  u.body = static_cast<uint32_t>((E.P[h.e] - u.Ps) + (E.QQ[h.s + (u.tl << E.ri_shift)] - u.Qs));
  return u;
}

template <int ENC>
__global__ void __launch_bounds__(ENC_THREADS, 4) k_encode_smem(EncView E, int S, const uint32_t* block_first, uint32_t nblocks,
                                                               const unsigned long long* block_off, uint8_t* out) {
  extern __shared__ __align__(16) uint8_t img_raw[];    // ENC_SMEM_CAP + 32
  __shared__ uint32_t tab0[256];
  __shared__ uint32_t stab[4][256];
  __shared__ uint32_t warp_crc[2];
  __shared__ uint32_t warp_sums[32];
  __shared__ unsigned long long t_src[ENC_EM_S];
  __shared__ uint32_t t_dsto[ENC_EM_S];
  __shared__ uint32_t t_len[ENC_EM_S];
  __shared__ uint32_t t_chunk[ENC_EM_S + 1];
  __shared__ uint16_t t_item[ENC_ITEMS_SMEM];
  static_assert(ENC_EM_S == ENC_THREADS && CRC_STRIDE_WORDS == ENC_THREADS, "one CRC lane per thread");
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) (&stab[0][0])[i] = (&g_crc_stride[0][0])[i];
  tab0[threadIdx.x] = g_crc_tab[0][threadIdx.x];
  // x^(32 * 4g): moves the fold of partials 4g .. 4g+3 to its distance from the end of the message
  const uint32_t crc_kc = g_crc_xpow8[16 * (threadIdx.x & 63)];
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;

  uint32_t b = blockIdx.x;
  EncBlkHdr nh{}; EncBlkSums ns{};
  if (b < nblocks) { nh = enc_load_hdr(E, block_first, block_off, b, nblocks); ns = enc_load_sums(E, nh); }
  for (; b < nblocks; b += gridDim.x) {
    const EncBlkHdr h = nh; const EncBlkSums u = ns;
    const uint32_t nb = b + gridDim.x;
    // the next block's parameters are fetched while this one is assembled
    if (nb < nblocks) nh = enc_load_hdr(E, block_first, block_off, nb, nblocks);
    if (h.btot > ENC_SMEM_CAP) {                                     // uniform for the CTA; k_encode_fused takes it
      if (nb < nblocks) ns = enc_load_sums(E, nh);
      continue;
    }
    const uint32_t blen = h.btot - 5;
    const uint32_t s = h.s, e = h.e;
    uint8_t* gdst = out + h.boff;
    // image[0] corresponds to gdst[0]; shifted so that image and destination agree mod 16
    const uint32_t mis = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(gdst) & 15);
    uint8_t* img = img_raw + mis;
    if (threadIdx.x < 4) reinterpret_cast<uint32_t*>(img_raw)[threadIdx.x] = 0;    // leading zeros do not change a CRC register of 0
    const unsigned long long Ps = u.Ps, Qs = u.Qs;
    const uint32_t tl = u.tl, body = u.body;
    __syncthreads();

    for (uint32_t p0 = s; p0 < e; p0 += ENC_EM_S) {
      const uint32_t pn = min(static_cast<uint32_t>(ENC_EM_S), e - p0);
      // ---- phase A: one thread per entry. Header + key delta bytes into the image, value copy job
      // into the table. All metadata loads of all entries are in flight together.
      for (uint32_t q = threadIdx.x; q < pn; q += blockDim.x) {
        const uint32_t j = p0 + q;
        const bool restart = ((j - s) & (E.ri - 1)) == 0;
        uint32_t off = static_cast<uint32_t>(E.P[j] - Ps);
        if (j > s) { const uint32_t tp = (j - 1 - s) >> E.ri_shift; off += static_cast<uint32_t>(E.QQ[s + (tp << E.ri_shift)] - Qs); }
        const Desc d = E.kept[j];
        const uint8_t* rec = kept_rec(E, d, S);
        const uint32_t vlen = d.vlen_out;
        const RunView& run = E.runs[d.run];
        const uint8_t* vs = run.data + run.val_off[d.gid - run.gid_base];
        uint8_t* p = emit_entry_key<ENC>(E, S, j, d, rec, kept_suffix(rec, d, S), restart, img + off);
        uint32_t copy_len = vlen;
        if (d.flags & ENT_VAL_TOMBSTONE) { p[0] = 'X'; copy_len = 0; }
        else if (d.flags & ENT_VAL_REENCODE) {
          const ValueRewrite& rw = E.rewrites[d.rewrite_slot];
          for (uint32_t i = 0; i < rw.prefix_len; i++) p[i] = rw.prefix[i];
          const uint32_t rest = vlen - rw.prefix_len;
          for (uint32_t i = 0; i < rest; i++) p[rw.prefix_len + i] = vs[rw.skip + i];
          copy_len = 0;
        }
        t_dsto[q] = static_cast<uint32_t>(p - img);
        t_src[q] = reinterpret_cast<unsigned long long>(vs);
        t_len[q] = copy_len;
        if (restart) {
          const uint32_t t = (j - s) >> E.ri_shift;
          uint8_t* r = img + body + 4 * t;
          r[0] = static_cast<uint8_t>(off); r[1] = static_cast<uint8_t>(off >> 8); r[2] = static_cast<uint8_t>(off >> 16); r[3] = static_cast<uint8_t>(off >> 24);
        }
      }
      __syncthreads();
      // items = destination-aligned 16-byte chunks of every value (image and HBM agree mod 16)
      uint32_t c0 = 0;
      {
        const uint32_t q0 = threadIdx.x;
        // number of 16-byte destination-aligned chunks lying entirely inside the value
        if (q0 < pn && t_len[q0]) {
          const uint32_t d0 = t_dsto[q0] + mis, d1 = d0 + t_len[q0];
          const uint32_t fa = (d0 + 15) & ~15u, fb = d1 & ~15u;
          c0 = fb > fa ? (fb - fa) >> 4 : 0;
        }
      }
      c0 = (c0 + 3) >> 2;                        // one item = up to four consecutive chunks of one value
      uint32_t total_items;
      const uint32_t ibase = block_exclusive_scan(c0, warp_sums, &total_items);
      t_chunk[threadIdx.x] = ibase;
      if (threadIdx.x == blockDim.x - 1) t_chunk[ENC_EM_S] = ibase + c0;
      __syncthreads();
      const bool direct = total_items <= ENC_ITEMS_SMEM;
      if (direct) {
        const uint32_t q = threadIdx.x;
        if (q < pn) for (uint32_t it = t_chunk[q]; it < t_chunk[q + 1]; it++) t_item[it] = static_cast<uint16_t>(q);
        __syncthreads();
      }
      // ---- phase B: value bytes. An item covers up to four destination-aligned 16-byte chunks and
      // needs at most five aligned source vectors, all fetched before the first store.
#pragma unroll 2
      for (uint32_t it = threadIdx.x; it < total_items; it += blockDim.x) {
        uint32_t q;
        if (direct) q = t_item[it];
        else {
          uint32_t lo = 0, hi = pn;
          while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (t_chunk[mid] <= it) lo = mid; else hi = mid; }
          q = lo;
        }
        // offsets below are relative to img_raw (16-byte aligned): r = image offset + mis
        const uint32_t d0 = t_dsto[q] + mis, d1 = d0 + t_len[q];
        const uint32_t A = ((d0 + 15) & ~15u) + 64u * (it - t_chunk[q]);
        const uint32_t nch = min(4u, ((d1 & ~15u) - A) >> 4);
        const uint8_t* src = reinterpret_cast<const uint8_t*>(t_src[q]) + (A - d0);
        const uint32_t sh = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(src) & 15);
        const uint4* sa = reinterpret_cast<const uint4*>(src - sh);
        const uint32_t nld = nch + (sh ? 1 : 0);
        uint4 v[5];
#pragma unroll
        for (int t = 0; t < 5; t++) v[t] = (static_cast<uint32_t>(t) < nld) ? __ldg(sa + t) : make_uint4(0, 0, 0, 0);
        uint4* dv = reinterpret_cast<uint4*>(img_raw + A);
#pragma unroll
        for (int t = 0; t < 4; t++) if (static_cast<uint32_t>(t) < nch) dv[t] = sh ? shift16(v[t], v[t + 1], sh) : v[t];
      }
      // value edges (bytes before the first / after the last full chunk): two small jobs per entry
      for (uint32_t t = threadIdx.x; t < 2 * pn; t += blockDim.x) {
        const uint32_t q = t >> 1;
        const uint32_t len = t_len[q];
        if (!len) continue;
        const uint32_t d0 = t_dsto[q] + mis, d1 = d0 + len;
        const uint32_t fa = (d0 + 15) & ~15u, fb = d1 & ~15u;
        uint32_t lo, hi;                           // byte range [lo, hi) of this edge, in img_raw offsets
        if (fb > fa) { if (t & 1) { lo = fb; hi = d1; } else { lo = d0; hi = fa; } }
        else { if (t & 1) continue; lo = d0; hi = d1; }          // short value: one job copies it all
        const uint8_t* src = reinterpret_cast<const uint8_t*>(t_src[q]) + (lo - d0);
        while (lo < hi) {
          const uint4 x = load_unaligned16(src);
          const uint32_t w[4] = {x.x, x.y, x.z, x.w};
          const uint32_t nbytes = min(16u, hi - lo);
#pragma unroll
          for (int bb = 0; bb < 16; bb++) if (bb < static_cast<int>(nbytes)) img_raw[lo + bb] = static_cast<uint8_t>(w[bb >> 2] >> (8 * (bb & 3)));
          lo += nbytes; src += nbytes;
        }
      }
      __syncthreads();
    }
    if (nb < nblocks) ns = enc_load_sums(E, nh);
    if (threadIdx.x == 0) {
      const uint32_t nres = tl + 1;
      uint8_t* q = img + body + 4 * nres;
      q[0] = static_cast<uint8_t>(nres); q[1] = static_cast<uint8_t>(nres >> 8); q[2] = static_cast<uint8_t>(nres >> 16); q[3] = static_cast<uint8_t>(nres >> 24);
      q[4] = 0;   // kNoCompression
    }
    __syncthreads();
    // ---- CRC32C over image[0, blen] from shared memory. The words of img_raw (zeros in front of
    // the image) are numbered from the END of the message; thread t owns the words at distance
    // t, t + 256, ... and folds them with the x^(8*1024) map, so consecutive lanes read consecutive
    // words and no per-thread polynomial shift is needed:
    //   R = sum_t T^(t+1) ( sum_j S^j w[t + 256 j] ),  T = one-word step, S = T^256.
    const uint32_t L = blen + 1;                                    // contents + type byte
    const uint32_t nwords = (mis + L) >> 2, tailb = (mis + L) & 3;
    {
      const uint32_t* wp = reinterpret_cast<const uint32_t*>(img_raw);
      // the 0xffffffff initial register == the first four message bytes complemented
      const uint32_t wi0 = mis >> 2, sh0 = (mis & 3) * 8;
      const uint32_t m0 = 0xffffffffu << sh0, m1 = sh0 ? 0xffffffffu >> (32 - sh0) : 0u;
      uint32_t acc = 0;
      if (nwords > threadIdx.x) {
        const uint32_t last = nwords - 1 - threadIdx.x;             // index of this thread's word nearest the end
        uint32_t i = last & (CRC_STRIDE_WORDS - 1);                 // its farthest word
        acc = wp[i];
        if (i == wi0) acc ^= m0; else if (i == wi0 + 1) acc ^= m1;
        for (i += CRC_STRIDE_WORDS; i <= last; i += CRC_STRIDE_WORDS) {
          acc = stab[3][acc & 0xff] ^ stab[2][(acc >> 8) & 0xff] ^ stab[1][(acc >> 16) & 0xff] ^ stab[0][acc >> 24];
          acc ^= wp[i];
        }
      }
      t_len[threadIdx.x] = acc;                                       // partial A_t (t_len is free by now)
    }
    __syncthreads();
    // R = sum_t T^(t+1) A_t. 64 threads take four consecutive partials each: four ordinary word steps
    // (byte table), then ONE multiplication by x^(32 * 4g) per thread — two warps instead of eight pay
    // for the bit-serial modular multiplication.
    if (threadIdx.x < 64) {
      uint32_t r = 0;
#pragma unroll
      for (int tp = 3; tp >= 0; tp--) {
        r ^= t_len[4 * threadIdx.x + tp];
#pragma unroll
        for (int q = 0; q < 4; q++) r = tab0[r & 0xff] ^ (r >> 8);
      }
      if (r) r = crc_mulmod(crc_kc, r);
      for (int o = 16; o; o >>= 1) r ^= __shfl_xor_sync(0xffffffffu, r, o);
      if (lane == 0) warp_crc[wid] = r;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t r = warp_crc[0] ^ warp_crc[1];
      const uint8_t* tp = img_raw + 4 * nwords;
      for (uint32_t i = 0; i < tailb; i++) r = tab0[(r ^ tp[i]) & 0xff] ^ (r >> 8);
      const uint32_t crc = crc_mask(~r);
      uint8_t* t = img + blen + 1;
      t[0] = static_cast<uint8_t>(crc); t[1] = static_cast<uint8_t>(crc >> 8); t[2] = static_cast<uint8_t>(crc >> 16); t[3] = static_cast<uint8_t>(crc >> 24);
    }
    __syncthreads();
    // ---- image -> HBM: 16-byte vector stores (image and destination agree mod 16)
    {
      const uint32_t total = h.btot;
      const uint32_t head = (16 - mis) & 15;
      const uint32_t hb = head < total ? head : total;
      if (threadIdx.x < hb) gdst[threadIdx.x] = img[threadIdx.x];
      const uint32_t nvec = (total - hb) >> 4;
      const uint4* sv = reinterpret_cast<const uint4*>(img + hb);
      uint4* dv = reinterpret_cast<uint4*>(gdst + hb);
      for (uint32_t v = threadIdx.x; v < nvec; v += blockDim.x) dv[v] = sv[v];
      const uint32_t done = hb + nvec * 16;
      if (threadIdx.x < total - done) gdst[done + threadIdx.x] = img[done + threadIdx.x];
    }
    __syncthreads();
  }
}

// ---- block assembler v4: value bytes never enter shared memory, the CRC never touches them ----------------
// Values are copied verbatim from the input files, and their RAW CRC32C is already known (RunView::val_crc, computed
// by the ingest pass while it verified the inputs). So
//   * the full destination-aligned 16-byte chunks of every value go global -> registers -> global (shifted into
//     place), without a stop in shared memory;
//   * shared memory holds only what is assembled byte by byte: entry headers, key deltas, the few value bytes
//     around chunk boundaries, rewritten values, the restart array and the trailer — the 16-byte chunks that
//     contain any such byte are stored from the image by the thread of the entry they begin in;
//   * the block checksum is the GF(2)-linear combination of per-entry pieces,
//       crc(block) = sum_e [ crc(gap_e) * x^(8 |value_e|) + crc(value_e) ] * x^(8 (L - end_e)) + crc(tail) + init term,
//     where gap_e = header + key delta of entry e, read from the image (a few dozen bytes per entry).
// Per 32 KB block that is ~2 modular multiplications and ~30 table look-ups per entry instead of four look-ups
// per 4 bytes of the whole image.
constexpr int ENC4_REP = 8;            // copies of the byte table (lane l uses copy l % 8)

template <int ENC>
__global__ void __launch_bounds__(ENC_THREADS, 4) k_encode_v4(EncView E, int S, const uint32_t* block_first, uint32_t nblocks,
                                                             const unsigned long long* block_off, uint8_t* out) {
  extern __shared__ __align__(16) uint8_t img_raw[];    // ENC_SMEM_CAP + 32
  __shared__ uint32_t tab0[256 * ENC4_REP];
  __shared__ uint32_t warp_sums[32];
  __shared__ unsigned long long t_src[ENC_EM_S];
  __shared__ uint32_t t_est[ENC_EM_S];      // entry start (image offset)
  __shared__ uint32_t t_dsto[ENC_EM_S];     // where the copied value body starts (image offset)
  __shared__ uint32_t t_len[ENC_EM_S];      // bytes copied from the input (0: the value was written into the image)
  __shared__ uint32_t t_end[ENC_EM_S];      // entry end (image offset)
  __shared__ uint32_t t_vcrc[ENC_EM_S];
  __shared__ uint32_t t_chunk[ENC_EM_S + 1];
  __shared__ uint16_t t_item[ENC_ITEMS_SMEM];
  __shared__ uint32_t sh_acc;
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    const uint32_t v = g_crc_tab[0][i];
#pragma unroll
    for (int c = 0; c < ENC4_REP; c++) tab0[i * ENC4_REP + c] = v;
  }
  const uint32_t copy = threadIdx.x & (ENC4_REP - 1);
  __syncthreads();
  const int lane = threadIdx.x & 31;

  uint32_t b = blockIdx.x;
  EncBlkHdr nh{}; EncBlkSums ns{};
  if (b < nblocks) { nh = enc_load_hdr(E, block_first, block_off, b, nblocks); ns = enc_load_sums(E, nh); }
  for (; b < nblocks; b += gridDim.x) {
    const EncBlkHdr h = nh; const EncBlkSums u = ns;
    const uint32_t nb = b + gridDim.x;
    if (nb < nblocks) nh = enc_load_hdr(E, block_first, block_off, nb, nblocks);
    if (h.btot > ENC_SMEM_CAP) {                                     // uniform for the CTA; k_encode_fused takes it
      if (nb < nblocks) ns = enc_load_sums(E, nh);
      continue;
    }
    const uint32_t blen = h.btot - 5;
    const uint32_t L = blen + 1;                                     // contents + type byte
    const uint32_t s = h.s, e = h.e;
    uint8_t* gdst = out + h.boff;
    const uint32_t mis = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(gdst) & 15);
    uint8_t* img = img_raw + mis;                                    // image and destination agree mod 16
    uint8_t* gbase = gdst - mis;                                     // 16-byte aligned; chunk c <-> img_raw[16c, 16c + 16)
    const uint32_t vlo = mis, vhi = mis + h.btot;                    // bytes of this block inside the chunk grid
    const unsigned long long Ps = u.Ps, Qs = u.Qs;
    const uint32_t tl = u.tl, body = u.body;
    if (threadIdx.x == 0) sh_acc = 0;
    // a chunk of the grid: whole chunks as one vector, the block's first / last partial chunk byte by byte
    auto store_chunk = [&](uint32_t c) {
      const uint32_t lo = 16 * c, hi = lo + 16;
      if (lo >= vlo && hi <= vhi) *reinterpret_cast<uint4*>(gbase + lo) = *reinterpret_cast<const uint4*>(img_raw + lo);
      else for (uint32_t x = max(lo, vlo); x < min(hi, vhi); x++) gbase[x] = img_raw[x];
    };
    __syncthreads();

    unsigned long long acc = 0;                  // XOR of unreduced carry-less products
    for (uint32_t p0 = s; p0 < e; p0 += ENC_EM_S) {
      const uint32_t pn = min(static_cast<uint32_t>(ENC_EM_S), e - p0);
      // ---- phase A: one thread per entry: header + key delta into the image, value copy job into the table
      for (uint32_t q = threadIdx.x; q < pn; q += blockDim.x) {
        const uint32_t j = p0 + q;
        const bool restart = ((j - s) & (E.ri - 1)) == 0;
        uint32_t off = static_cast<uint32_t>(E.P[j] - Ps);
        if (j > s) { const uint32_t tp = (j - 1 - s) >> E.ri_shift; off += static_cast<uint32_t>(E.QQ[s + (tp << E.ri_shift)] - Qs); }
        const Desc d = E.kept[j];
        const uint8_t* rec = kept_rec(E, d, S);
        const uint32_t vlen = d.vlen_out;
        const RunView& run = E.runs[d.run];
        const uint32_t idx = d.gid - run.gid_base;
        const uint8_t* vs = run.data + run.val_off[idx];
        uint8_t* p = emit_entry_key<ENC>(E, S, j, d, rec, kept_suffix(rec, d, S), restart, img + off);
        uint32_t copy_len = vlen;
        uint32_t vcrc = 0;
        if (d.flags & ENT_VAL_TOMBSTONE) { p[0] = 'X'; copy_len = 0; }
        else if (d.flags & ENT_VAL_REENCODE) {
          const ValueRewrite& rw = E.rewrites[d.rewrite_slot];
          for (uint32_t i = 0; i < rw.prefix_len; i++) p[i] = rw.prefix[i];
          const uint32_t rest = vlen - rw.prefix_len;
          for (uint32_t i = 0; i < rest; i++) p[rw.prefix_len + i] = vs[rw.skip + i];
          copy_len = 0;
        } else if (vlen) vcrc = run.val_crc[idx];
        t_est[q] = off + mis;
        t_dsto[q] = static_cast<uint32_t>(p - img_raw);
        t_end[q] = static_cast<uint32_t>(p - img_raw) + vlen;
        t_src[q] = reinterpret_cast<unsigned long long>(vs);
        t_len[q] = copy_len;
        t_vcrc[q] = vcrc;
        if (restart) {
          const uint32_t t = (j - s) >> E.ri_shift;
          uint8_t* r = img + body + 4 * t;
          r[0] = static_cast<uint8_t>(off); r[1] = static_cast<uint8_t>(off >> 8); r[2] = static_cast<uint8_t>(off >> 16); r[3] = static_cast<uint8_t>(off >> 24);
        }
      }
      __syncthreads();
      // items = runs of up to four destination-aligned 16-byte chunks lying entirely inside one value
      uint32_t c0 = 0;
      {
        const uint32_t q0 = threadIdx.x;
        if (q0 < pn && t_len[q0]) {
          const uint32_t d0 = t_dsto[q0], d1 = d0 + t_len[q0];
          const uint32_t fa = (d0 + 15) & ~15u, fb = d1 & ~15u;
          c0 = fb > fa ? (fb - fa) >> 4 : 0;
        }
      }
      c0 = (c0 + 3) >> 2;
      uint32_t total_items;
      const uint32_t ibase = block_exclusive_scan(c0, warp_sums, &total_items);
      t_chunk[threadIdx.x] = ibase;
      if (threadIdx.x == blockDim.x - 1) t_chunk[ENC_EM_S] = ibase + c0;
      __syncthreads();
      const bool direct = total_items <= ENC_ITEMS_SMEM;
      if (direct) {
        const uint32_t q = threadIdx.x;
        if (q < pn) for (uint32_t it = t_chunk[q]; it < t_chunk[q + 1]; it++) t_item[it] = static_cast<uint16_t>(q);
        __syncthreads();
      }
      // ---- phase B: value bodies, HBM -> registers -> HBM
#pragma unroll 2
      for (uint32_t it = threadIdx.x; it < total_items; it += blockDim.x) {
        uint32_t q;
        if (direct) q = t_item[it];
        else {
          uint32_t lo = 0, hi = pn;
          while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (t_chunk[mid] <= it) lo = mid; else hi = mid; }
          q = lo;
        }
        const uint32_t d0 = t_dsto[q], d1 = d0 + t_len[q];
        const uint32_t A = ((d0 + 15) & ~15u) + 64u * (it - t_chunk[q]);
        const uint32_t nch = min(4u, ((d1 & ~15u) - A) >> 4);
        const uint8_t* src = reinterpret_cast<const uint8_t*>(t_src[q]) + (A - d0);
        const uint32_t sh = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(src) & 15);
        const uint4* sa = reinterpret_cast<const uint4*>(src - sh);
        const uint32_t nld = nch + (sh ? 1 : 0);
        uint4 v[5];
#pragma unroll
        for (int t = 0; t < 5; t++) v[t] = (static_cast<uint32_t>(t) < nld) ? __ldg(sa + t) : make_uint4(0, 0, 0, 0);
        uint4* dv = reinterpret_cast<uint4*>(gbase + A);
#pragma unroll
        for (int t = 0; t < 4; t++) if (static_cast<uint32_t>(t) < nch) dv[t] = sh ? shift16(v[t], v[t + 1], sh) : v[t];
      }
      // value edges (bytes before the first / after the last full chunk) into the image: two small jobs per entry
      for (uint32_t t = threadIdx.x; t < 2 * pn; t += blockDim.x) {
        const uint32_t q = t >> 1;
        const uint32_t len = t_len[q];
        if (!len) continue;
        const uint32_t d0 = t_dsto[q], d1 = d0 + len;
        const uint32_t fa = (d0 + 15) & ~15u, fb = d1 & ~15u;
        uint32_t lo, hi;
        if (fb > fa) { if (t & 1) { lo = fb; hi = d1; } else { lo = d0; hi = fa; } }
        else { if (t & 1) continue; lo = d0; hi = d1; }
        const uint8_t* src = reinterpret_cast<const uint8_t*>(t_src[q]) + (lo - d0);
        while (lo < hi) {
          const uint4 x = load_unaligned16(src);
          const uint32_t w[4] = {x.x, x.y, x.z, x.w};
          const uint32_t nbytes = min(16u, hi - lo);
#pragma unroll
          for (int bb = 0; bb < 16; bb++) if (bb < static_cast<int>(nbytes)) img_raw[lo + bb] = static_cast<uint8_t>(w[bb >> 2] >> (8 * (bb & 3)));
          lo += nbytes; src += nbytes;
        }
      }
      __syncthreads();
      // ---- phase C: per entry, its share of the block checksum and the chunks it owns
      for (uint32_t q = threadIdx.x; q < pn; q += blockDim.x) {
        const uint32_t est = t_est[q], d0 = t_dsto[q], len = t_len[q], eend = t_end[q];
        const uint32_t fa = (d0 + 15) & ~15u, fb = (d0 + len) & ~15u;
        const bool full = len && fb > fa;
        // checksum: the bytes that exist only in the image are the entry's "gap" (a rewritten value belongs to it);
        // a short copied value (no full chunk) sits in the image as well, but its CRC is known
        const uint32_t gap_end = len ? d0 : eend;
        uint32_t gc = 0;
        for (uint32_t x = est; x < gap_end; x++) gc = tab0[((gc ^ img_raw[x]) & 0xff) * ENC4_REP + copy] ^ (gc >> 8);
        // gap * x^(8 (bytes behind the gap)) + value * x^(8 (bytes behind the value)), unreduced
        acc ^= crc_clmul(gc, __ldg(&g_crc_xpow8[(mis + L) - gap_end]));
        if (len) acc ^= crc_clmul(t_vcrc[q], __ldg(&g_crc_xpow8[(mis + L) - eend]));
        // chunks: from the one the entry starts in up to the first full value chunk (or the end of the entry)
        const uint32_t c_lo = est >> 4, c_hi = full ? (fa >> 4) : ((eend + 15) >> 4);
        for (uint32_t c = c_lo; c < c_hi; c++) store_chunk(c);
      }
      __syncthreads();
    }
    if (nb < nblocks) ns = enc_load_sums(E, nh);
    // ---- tail: restart count + type byte, checksum, trailer, the chunks behind the last entry
    if (threadIdx.x == 0) {
      const uint32_t nres = tl + 1;
      uint8_t* q = img + body + 4 * nres;
      q[0] = static_cast<uint8_t>(nres); q[1] = static_cast<uint8_t>(nres >> 8); q[2] = static_cast<uint8_t>(nres >> 16); q[3] = static_cast<uint8_t>(nres >> 24);
      q[4] = 0;   // kNoCompression
    }
    {
      uint32_t a32 = crc_clmul_reduce(acc, [&](uint32_t x) { return tab0[x * ENC4_REP + copy]; });
      a32 = __reduce_xor_sync(0xffffffffu, a32);
      if (lane == 0 && a32) atomicXor(&sh_acc, a32);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t r = sh_acc, tc = 0;
      for (uint32_t x = body; x < L; x++) tc = tab0[((tc ^ img[x]) & 0xff) * ENC4_REP + copy] ^ (tc >> 8);
      r ^= tc;
      r ^= crc_mulmod(__ldg(&g_crc_xpow8[L]), 0xffffffffu);        // the 0xffffffff initial register, L <= 36 K
      const uint32_t crc = crc_mask(~r);
      uint8_t* t = img + blen + 1;
      t[0] = static_cast<uint8_t>(crc); t[1] = static_cast<uint8_t>(crc >> 8); t[2] = static_cast<uint8_t>(crc >> 16); t[3] = static_cast<uint8_t>(crc >> 24);
    }
    __syncthreads();
    {
      const uint32_t c_lo = (mis + body) >> 4, c_hi = (vhi + 15) >> 4;
      for (uint32_t c = c_lo + threadIdx.x; c < c_hi; c += blockDim.x) store_chunk(c);
    }
    __syncthreads();
  }
}

// ---- warp-per-block assembler (v5) ---------------------------------------------------------------
// One WARP builds one output block; nothing in the kernel waits on a CTA-wide barrier and there is no block image:
//   * a lane owns an entry: it writes the bytes that exist nowhere else — header + key delta, a tombstone's 'X', the
//     prefix of a rewritten value (the entry's "gap") — into its private scratch row, END-aligned to a word (its
//     length is known beforehand from nr / D) behind zero padding: the gap's raw CRC is then a handful of whole-word
//     table steps (leading zeros do not move a zero register);
//   * the warp then walks the round's entries two at a time, one per half-warp: the gap goes scratch -> HBM, the value
//     HBM -> registers -> HBM as destination-aligned 16-byte chunks (one per lane, two aligned source vectors funnel-
//     shifted into place), the <= 15 bytes in front of the first / behind the last full chunk as one byte per lane;
//     each step's value loads are issued one step ahead of its stores;
//   * the block checksum is the same GF(2)-linear combination as in v4 — every gap, value and restart-array word
//     enters as (raw CRC) * x^(8 * bytes behind it), XOR-accumulated unreduced per lane — so no byte of the block is
//     read back.
// Shared memory per CTA: the four slicing tables (4 KB) + one scratch row per lane, which leaves the occupancy to the
// register file (v4: one 36 KB image per CTA, four CTAs per SM, seven CTA barriers per block). Blocks of any size.
constexpr int ENC5_THREADS = 256;
__device__ __forceinline__ uint32_t enc5_crc_word(const uint32_t (*tab)[256], uint32_t c, uint32_t w) {
  c ^= w;
  return tab[3][c & 0xff] ^ tab[2][(c >> 8) & 0xff] ^ tab[1][(c >> 16) & 0xff] ^ tab[0][c >> 24];
}
__device__ __forceinline__ uint32_t enc5_xpow(unsigned long long nbytes) {
  return nbytes <= CRC_XPOW_TABLE ? __ldg(&g_crc_xpow8[nbytes]) : crc_xpow_bytes(nbytes, g_crc_x2n);
}
__device__ __forceinline__ void enc5_prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ void enc5_store_u32(uint8_t* p, uint32_t v) {
  p[0] = static_cast<uint8_t>(v); p[1] = static_cast<uint8_t>(v >> 8); p[2] = static_cast<uint8_t>(v >> 16); p[3] = static_cast<uint8_t>(v >> 24);
}

// One walk step of a half-warp: lane hl's share of a copied value (vd = its destination, len bytes from src). Loads:
// the first destination-aligned 16-byte chunk of the lane (two aligned source vectors, funnel-shifted at the store),
// one byte in front of the first / behind the last full chunk (a value without a full chunk: bytes hl and hl + 16).
// enc5_put stores them, and the further chunks of a value longer than 16 chunks.
struct Enc5Pre { uint4 a, b; uint32_t x; };          // x = source shift | head byte << 8 | tail byte << 16
__device__ __forceinline__ Enc5Pre enc5_fetch(const uint8_t* vd, const uint8_t* src, uint32_t len, uint32_t hl) {
  Enc5Pre t;
  t.a = make_uint4(0, 0, 0, 0); t.b = t.a;
  uint32_t sh = 0, hb = 0, tb = 0;
  if (len) {
    const uintptr_t d0 = reinterpret_cast<uintptr_t>(vd), d1 = d0 + len;
    const uintptr_t fa = (d0 + 15) & ~static_cast<uintptr_t>(15), fb = d1 & ~static_cast<uintptr_t>(15);
    if (fb > fa) {
      if (d0 + hl < fa) hb = __ldg(src + hl);
      if (fb + hl < d1) tb = __ldg(src + (fb - d0) + hl);
      const uintptr_t A = fa + 16u * hl;
      if (A < fb) {
        const uint8_t* s = src + (A - d0);
        sh = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(s) & 15);
        const uint4* v = reinterpret_cast<const uint4*>(s - sh);
        t.a = __ldg(v);
        if (sh) t.b = __ldg(v + 1);
      }
    } else {
      if (hl < len) hb = __ldg(src + hl);
      if (hl + 16 < len) tb = __ldg(src + hl + 16);
    }
  }
  t.x = sh | (hb << 8) | (tb << 16);
  return t;
}
__device__ __forceinline__ void enc5_put(const Enc5Pre& t, uint8_t* vd, const uint8_t* src, uint32_t len, uint32_t hl) {
  if (!len) return;
  const uint8_t hb = static_cast<uint8_t>(t.x >> 8), tb = static_cast<uint8_t>(t.x >> 16);
  const uintptr_t d0 = reinterpret_cast<uintptr_t>(vd), d1 = d0 + len;
  const uintptr_t fa = (d0 + 15) & ~static_cast<uintptr_t>(15), fb = d1 & ~static_cast<uintptr_t>(15);
  if (fb > fa) {
    if (d0 + hl < fa) vd[hl] = hb;
    if (fb + hl < d1) *reinterpret_cast<uint8_t*>(fb + hl) = tb;
    uintptr_t A = fa + 16u * hl;
    if (A < fb) {
      const uint32_t sh = t.x & 15;
      *reinterpret_cast<uint4*>(A) = sh ? shift16(t.a, t.b, sh) : t.a;
      for (A += 256; A < fb; A += 256) copy_chunk16(reinterpret_cast<uint8_t*>(A), src + (A - d0));
    }
  } else {
    if (hl < len) vd[hl] = hb;
    if (hl + 16 < len) vd[hl + 16] = tb;
  }
}

template <int ENC>
__global__ void __launch_bounds__(ENC5_THREADS, ENC == 1 ? 4 : 2) k_encode_v5(EncView E, int S, const uint32_t* block_first, uint32_t nblocks,
                                                          const unsigned long long* block_off, uint8_t* out, uint32_t G) {
  extern __shared__ __align__(16) uint8_t v5_smem[];      // tab[4][256], then ENC5_THREADS scratch rows of G bytes
  uint32_t (*tab)[256] = reinterpret_cast<uint32_t (*)[256]>(v5_smem);
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) (&tab[0][0])[i] = (&g_crc_tab[0][0])[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, hl = lane & 15, half = lane >> 4;
  uint8_t* const wsc = v5_smem + 4096 + static_cast<uint32_t>(wid) * 32u * G;
  uint8_t* const sc = wsc + static_cast<uint32_t>(lane) * G;      // G = an odd number of words: the lanes' rows start in different banks
  const uint32_t nwarps = gridDim.x * (ENC5_THREADS / 32);
  for (uint32_t b = blockIdx.x * (ENC5_THREADS / 32) + wid; b < nblocks; b += nwarps) {
    const unsigned long long boff = block_off[b];
    const unsigned long long L = block_off[b + 1] - boff - 4;          // contents + type byte
    const uint32_t s = block_first[b], e = (b + 1 < nblocks) ? block_first[b + 1] : E.n;
    const unsigned long long Ps = E.P[s];
    const unsigned long long Qs = E.QQ[s] - static_cast<unsigned long long>(static_cast<long long>(E.D[s]));
    const uint32_t tl = (e - 1 - s) >> E.ri_shift;
    const unsigned long long body = (E.P[e] - Ps) + (E.QQ[s + (tl << E.ri_shift)] - Qs);
    uint8_t* const blk = out + boff;
    unsigned long long acc = 0;                  // XOR of unreduced carry-less products
    // The kernel is bound by memory latency (a round's loads form a chain: descriptor -> record / value offset -> value
    // bytes), so the next round's chain is started ahead: its descriptors are loaded while this round's entries are
    // assembled, its record lines are requested into L2 while this round's values are copied. Its value lines are not:
    // with every warp of the machine asking for the next 32 values (~43 MB ahead, most of the 50 MB L2, which also holds
    // the lines being written) part of them was evicted before use and read from DRAM twice (DESIGN.md §4).
    Desc d_cur{};
    if (s + lane < e) d_cur = E.kept[s + lane];
    for (uint32_t r0 = s; r0 < e; r0 += 32) {
      const uint32_t j = r0 + lane;
      const uint32_t jn = j + 32;
      Desc d_next{};
      if (jn < e) d_next = E.kept[jn];
      unsigned long long eoff = 0, srcp = 0;
      uint32_t gap_len = 0, copy_len = 0;
      if (j < e) {
        const bool restart = ((j - s) & (E.ri - 1)) == 0;
        eoff = E.P[j] - Ps;
        if (j > s) { const uint32_t tp = (j - 1 - s) >> E.ri_shift; eoff += E.QQ[s + (tp << E.ri_shift)] - Qs; }
        const Desc d = d_cur;
        const uint8_t* rec = kept_rec(E, d, S);
        const RunView& run = E.runs[d.run];
        const uint32_t idx = d.gid - run.gid_base;
        const uint8_t* vs = run.data + run.val_off[idx];
        const uint32_t vlen = d.vlen_out;
        uint32_t esize = E.nr[j];
        if (restart) esize += static_cast<uint32_t>(static_cast<int32_t>(E.D[j]));
        const ValueRewrite* rw = nullptr;
        copy_len = vlen;
        if (d.flags & ENT_VAL_TOMBSTONE) copy_len = 0;
        else if (d.flags & ENT_VAL_REENCODE) { rw = &E.rewrites[d.rewrite_slot]; copy_len = vlen - rw->prefix_len; vs += rw->skip; }
        gap_len = esize - copy_len;
        const uint32_t pad = (4u - (gap_len & 3u)) & 3u;
        *reinterpret_cast<uint32_t*>(sc) = 0;
        uint8_t* p = emit_entry_key<ENC>(E, S, j, d, rec, kept_suffix(rec, d, S), restart, sc + pad);
        if (d.flags & ENT_VAL_TOMBSTONE) *p++ = 'X';
        else if (rw) for (uint32_t i = 0; i < rw->prefix_len; i++) *p++ = rw->prefix[i];
        uint32_t vcrc = 0;
        if (copy_len) {
          if (rw) { for (uint32_t i = 0; i < copy_len; i++) vcrc = tab[0][(vcrc ^ __ldg(vs + i)) & 0xff] ^ (vcrc >> 8); }
          else vcrc = run.val_crc[idx];
        }
        uint32_t gc = 0;
        const uint32_t* w = reinterpret_cast<const uint32_t*>(sc);
        const uint32_t nw = (pad + gap_len) >> 2;
        for (uint32_t i = 0; i < nw; i++) gc = enc5_crc_word(tab, gc, w[i]);
        const unsigned long long gap_end = eoff + gap_len;
        acc ^= crc_clmul(gc, enc5_xpow(L - gap_end));
        if (copy_len) acc ^= crc_clmul(vcrc, enc5_xpow(L - gap_end - copy_len));
        srcp = reinterpret_cast<unsigned long long>(vs);
        if (restart) {
          const uint32_t t = (j - s) >> E.ri_shift;
          const uint32_t o32 = static_cast<uint32_t>(eoff);
          enc5_store_u32(blk + body + 4ull * t, o32);
          acc ^= crc_clmul(enc5_crc_word(tab, 0u, o32), enc5_xpow(L - (body + 4ull * t + 4)));
        }
      }
      __syncwarp();
      if (jn < e) {
        const RunView& rn = E.runs[d_next.run];
        enc5_prefetch_l2(rn.rec + static_cast<size_t>(d_next.gid - rn.gid_base) * S);
      }
      // The warp walks the round's entries two at a time, one per half-warp, software-pipelined: the value loads of the
      // next step are issued before this step's stores, so that a step's stores wait on no load of their own (a 64-
      // register budget holds one step ahead; two ahead spill and were slower).
      const uint32_t nact = min(32u, e - r0);
      const uint32_t nsteps = (nact + 1) >> 1;
      auto step_args = [&](uint32_t st, uint8_t*& gdst, const uint8_t*& src, uint32_t& gap, uint32_t& len) {
        const uint32_t q = 2 * st + half;
        const unsigned long long eoff_q = __shfl_sync(0xffffffffu, eoff, q & 31);
        src = reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, srcp, q & 31));
        gap = __shfl_sync(0xffffffffu, gap_len, q & 31);
        len = __shfl_sync(0xffffffffu, copy_len, q & 31);
        gdst = blk + eoff_q;
        if (q >= nact) { gap = 0; len = 0; }
      };
      Enc5Pre pre;
      {
        uint8_t* gdst; const uint8_t* src; uint32_t gap, len;
        step_args(0, gdst, src, gap, len);
        pre = enc5_fetch(gdst + gap, src, len, hl);
      }
      for (uint32_t st = 0; st < nsteps; st++) {
        uint8_t* gdst; const uint8_t* src; uint32_t gap, len;
        step_args(st + 1, gdst, src, gap, len);
        const Enc5Pre nx = enc5_fetch(gdst + gap, src, st + 1 < nsteps ? len : 0u, hl);
        step_args(st, gdst, src, gap, len);
        const uint8_t* scq = wsc + (2 * st + half) * G + ((4u - (gap & 3u)) & 3u);
        if (hl < gap) gdst[hl] = scq[hl];
        if (hl + 16 < gap) gdst[hl + 16] = scq[hl + 16];
        for (uint32_t i = hl + 32; i < gap; i += 16) gdst[i] = scq[i];
        enc5_put(pre, gdst + gap, src, len, hl);
        pre = nx;
      }
      d_cur = d_next;
      __syncwarp();                                // the scratch rows are rewritten by the next round
    }
    // restart count + type byte, the 0xffffffff initial register's share, trailer
    uint32_t a32 = crc_clmul_reduce(acc, [&](uint32_t x) { return tab[0][x]; });
    a32 = __reduce_xor_sync(0xffffffffu, a32);
    if (lane == 0) {
      const uint32_t nres = tl + 1;
      uint8_t* q = blk + body + 4ull * nres;
      enc5_store_u32(q, nres);
      q[4] = 0;   // kNoCompression
      uint32_t tc = enc5_crc_word(tab, 0u, nres);
      tc = tab[0][tc & 0xff] ^ (tc >> 8);                                // the type byte (0)
      const uint32_t r = a32 ^ tc ^ crc_clmul_reduce(crc_clmul(enc5_xpow(L), 0xffffffffu), [&](uint32_t x) { return tab[0][x]; });
      enc5_store_u32(blk + L, crc_mask(~r));
    }
  }
}

// ---- bloom filter blocks (block_based_table_builder.cc:514-528,594-620; util/bloom.cc:43-61,384-455) ----
// One thread per distinct filter key (new_entry[ord] = survivor that introduces it): hash it and set
// its bits in filter block ord / max_keys. All probes of a key fall into one 64-byte line.
__global__ void __launch_bounds__(256) k_filter_build(EncView E, int S, const uint32_t* new_entry, uint32_t n_keys, BloomGeometry g, uint8_t* filters) {
  for (uint32_t ord = blockIdx.x * blockDim.x + threadIdx.x; ord < n_keys; ord += gridDim.x * blockDim.x) {
    const uint32_t j = new_entry[ord];
    const Desc d = E.kept[j];
    const uint8_t* rec = kept_rec(E, d, S);
    uint32_t h = leveldb_hash(rec, E.fk_len[j], kBloomSeed);
    const uint32_t delta = (h >> 17) | (h << 15);
    uint32_t* line = reinterpret_cast<uint32_t*>(filters + static_cast<size_t>(ord / g.max_keys) * g.dev_stride) + (h % g.num_lines) * (kBloomLineBits / 32);
    for (uint32_t i = 0; i < g.num_probes; i++) {
      const uint32_t bit = h % kBloomLineBits;
      atomicOr(line + (bit >> 5), 1u << (bit & 31));
      h += delta;
    }
  }
}

// Same, one CTA per filter block with the bits assembled in shared memory (a 64 KB block fits):
// shared-memory atomics instead of ~6 scattered global atomics per key, then one coalesced write.
constexpr uint32_t FILTER_SMEM_MAX = 96 * 1024;
__global__ void __launch_bounds__(1024) k_filter_build_smem(const uint32_t* hashes, uint32_t n_keys, BloomGeometry g, uint32_t nfb,
                                                            uint32_t parts, uint8_t* filters) {
  // `parts` CTAs share one filter block (each takes a slice of its keys); the zero-initialised
  // global block receives the non-zero words of every partial image by atomicOr.
  extern __shared__ __align__(16) uint32_t fbits[];
  const uint32_t words = g.dev_stride / 4;
  for (uint32_t t = blockIdx.x; t < nfb * parts; t += gridDim.x) {
    const uint32_t f = t / parts, part = t - f * parts;
    for (uint32_t i = threadIdx.x; i < words; i += blockDim.x) fbits[i] = 0;
    __syncthreads();
    const uint32_t lo = f * g.max_keys, hi = min(n_keys, lo + g.max_keys);
    const uint32_t per = (hi - lo + parts - 1) / parts;
    const uint32_t plo = min(hi, lo + part * per), phi = min(hi, plo + per);
    for (uint32_t ord = plo + threadIdx.x; ord < phi; ord += blockDim.x) {
      uint32_t h = hashes[ord];
      const uint32_t delta = (h >> 17) | (h << 15);
      uint32_t* line = fbits + (h % g.num_lines) * (kBloomLineBits / 32);
      for (uint32_t i = 0; i < g.num_probes; i++) {
        const uint32_t bit = h % kBloomLineBits;
        atomicOr(line + (bit >> 5), 1u << (bit & 31));
        h += delta;
      }
    }
    __syncthreads();
    uint32_t* out = reinterpret_cast<uint32_t*>(filters + static_cast<size_t>(f) * g.dev_stride);
    if (parts == 1) { for (uint32_t i = threadIdx.x; i < words; i += blockDim.x) out[i] = fbits[i]; }
    else { for (uint32_t i = threadIdx.x; i < words; i += blockDim.x) if (fbits[i]) atomicOr(out + i, fbits[i]); }
    __syncthreads();
  }
}

// Per filter block: metadata bytes, and for the host-side filter index the last key added to the
// block and the first key of the block ([u16 len][bytes], stride KB each).
__global__ void __launch_bounds__(256) k_filter_finish(EncView E, int S, const uint32_t* new_entry, uint32_t n_keys, BloomGeometry g, uint32_t nfb,
                                                       uint8_t* filters, uint8_t* keys_out, uint32_t KB, uint32_t* first_entry) {
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < nfb * 2; t += gridDim.x * blockDim.x) {
    const uint32_t f = t >> 1, which = t & 1;
    uint8_t* o = keys_out + static_cast<size_t>(t) * KB;
    const uint32_t lo = f * g.max_keys;
    if (lo >= n_keys) { o[0] = 0; o[1] = 0; if (!which) first_entry[f] = 0; }
    else {
      const uint32_t hi = min(n_keys, lo + g.max_keys);
      const uint32_t j = new_entry[which ? hi - 1 : lo];
      if (!which) first_entry[f] = j;
      const uint32_t fl = E.fk_len[j];
      const uint8_t* rec = kept_rec(E, E.kept[j], S);
      o[0] = static_cast<uint8_t>(fl); o[1] = static_cast<uint8_t>(fl >> 8);
      for (uint32_t q = 0; q < fl; q++) o[2 + q] = rec[q];
    }
    if (!which) {
      uint8_t* meta = filters + static_cast<size_t>(f) * g.dev_stride + (g.block_bytes - 5);
      meta[0] = static_cast<uint8_t>(g.num_probes);
      for (int q = 0; q < 4; q++) meta[1 + q] = static_cast<uint8_t>(g.num_lines >> (8 * q));
    }
  }
}

// Boundary keys for the host-side index: for every block its last internal key and the first key
// of the next block, fixed stride KB bytes each: [u16 len][bytes].
__global__ void __launch_bounds__(256) k_boundary_keys(EncView E, int S, const uint32_t* block_first, uint32_t nblocks, uint8_t* out, uint32_t KB) {
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < nblocks * 2 + 1; t += gridDim.x * blockDim.x) {
    const uint32_t b = t >> 1, which = t & 1;
    const uint32_t e = (b + 1 < nblocks) ? block_first[b + 1] : E.n;
    uint8_t* o = out + static_cast<size_t>(t) * KB;
    const uint32_t j = b == nblocks ? 0u : (which ? e : e - 1);      // the extra slot: the first key of the file
    if (j >= E.n) { o[0] = 0; o[1] = 0; continue; }
    const Desc d = E.kept[j];
    const uint8_t* rec = kept_rec(E, d, S);
    const uint32_t ulen = d.klen - 8u;
    o[0] = static_cast<uint8_t>(d.klen); o[1] = static_cast<uint8_t>(d.klen >> 8);
    for (uint32_t q = 0; q < ulen; q++) o[2 + q] = rec[q];
    const uint64_t suffix = kept_suffix(rec, d, S);
    for (int q = 0; q < 8; q++) o[2 + ulen + q] = static_cast<uint8_t>(suffix >> (8 * q));
  }
}


// ---- FileMetaData user boundary values (a19) --------------------------------------------------------------------
// DocDBCompactionFeed::UpdateBoundaryValues (docdb_compaction_context.cc:754-773) feeds the first entry it passes on
// for every DocKey to DocBoundaryValuesExtractor::Extract (doc_boundary_values_extractor.cc:40-64): the encoded
// range-group components of the DocKey (hashed components are not reported, internal meta records are skipped),
// tag = 10 + component index, and keeps per tag the bytewise smallest and largest value (rocksdb/db/metadata.cc:44-57).
// Here: the survivors that carry ENT_FIRST_OF_ROW are walked once; every thread keeps (pointer, length) of its best
// candidates per component, warps and CTAs reduce them by comparing the bytes behind the pointers, the last kernel
// copies the winners out.
constexpr int BV_MAXC = 16;            // range components reported (tags 10 .. 25)
constexpr int BV_MAXLEN = 255;         // longest component value copied out
struct BvCand { const uint8_t* p; uint32_t len; uint32_t valid; };
struct BvOut { uint32_t n_comps; uint32_t overflow; uint32_t len[2][BV_MAXC]; uint8_t val[2][BV_MAXC][BV_MAXLEN + 1]; };

__device__ __forceinline__ int bv_cmp(const uint8_t* a, uint32_t la, const uint8_t* b, uint32_t lb) {
  const uint32_t m = la < lb ? la : lb;
  for (uint32_t i = 0; i < m; i++) { const uint8_t x = a[i], y = b[i]; if (x != y) return x < y ? -1 : 1; }
  return la < lb ? -1 : (la > lb ? 1 : 0);
}
// which = 0: keep the smaller, 1: keep the larger
__device__ __forceinline__ void bv_take(BvCand* best, const uint8_t* p, uint32_t len, int which) {
  if (!best->valid) { best->p = p; best->len = len; best->valid = 1; return; }
  const int c = bv_cmp(p, len, best->p, best->len);
  if (which == 0 ? c < 0 : c > 0) { best->p = p; best->len = len; }
}

__global__ void __launch_bounds__(256) k_boundary_values(EncView E, int S, BvCand* cand /*[grid][2][BV_MAXC]*/, BvOut* out) {
  BvCand best[2][BV_MAXC];
#pragma unroll
  for (int w = 0; w < 2; w++)
    for (int c = 0; c < BV_MAXC; c++) { best[w][c].p = nullptr; best[w][c].len = 0; best[w][c].valid = 0; }
  uint32_t ncomp = 0;
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < E.n; j += gridDim.x * blockDim.x) {
    const Desc d = E.kept[j];
    if (!(d.flags & ENT_FIRST_OF_ROW)) continue;
    const uint8_t* key = kept_rec(E, d, S);
    const int ulen = static_cast<int>(d.klen) - 8;
    if (ulen <= 0) continue;
    const uint8_t t0 = key[0];
    if (t0 == 6 || t0 == 7 || t0 == 8 || t0 == 'x') continue;          // IsMetaKeyType (dockv/value_type.h:252-273)
    int pos = dockey_id_size(key, ulen);
    if (pos < 0) continue;
    if (pos < ulen && key[pos] == 'G') {                                 // hash code + hashed group: not reported
      if (ulen - pos < 3) continue;
      pos += 3;
      const int k = consume_primitive_group(key + pos, ulen - pos);
      if (k < 0) continue;
      pos += k;
    }
    uint32_t c = 0;
    while (pos < ulen && key[pos] != '!') {
      if (is_special_key_entry_type(key[pos])) break;
      const int k = key_entry_size(key + pos, ulen - pos);
      if (k < 0) break;
      if (c < BV_MAXC) { bv_take(&best[0][c], key + pos, k, 0); bv_take(&best[1][c], key + pos, k, 1); }
      else out->overflow = 1;
      pos += k; c++;
    }
    ncomp = max(ncomp, min(c, static_cast<uint32_t>(BV_MAXC)));
  }
  // CTA reduction, component by component (only as many as any thread of the CTA has seen)
  __shared__ BvCand sh[2][8];
  __shared__ uint32_t sh_nc;
  if (threadIdx.x == 0) sh_nc = 0;
  __syncthreads();
  if (ncomp) atomicMax(&sh_nc, ncomp);
  __syncthreads();
  const uint32_t nc = sh_nc;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (uint32_t c = 0; c < nc; c++) {
#pragma unroll
    for (int w = 0; w < 2; w++) {
      BvCand b = best[w][c];
      for (int o = 16; o; o >>= 1) {
        BvCand y;
        y.p = reinterpret_cast<const uint8_t*>(__shfl_xor_sync(0xffffffffu, reinterpret_cast<unsigned long long>(b.p), o));
        y.len = __shfl_xor_sync(0xffffffffu, b.len, o);
        y.valid = __shfl_xor_sync(0xffffffffu, b.valid, o);
        if (y.valid) bv_take(&b, y.p, y.len, w);
      }
      if (lane == 0) sh[w][wid] = b;
    }
    __syncthreads();
    if (threadIdx.x < 2) {
      const int w = threadIdx.x;
      BvCand b = sh[w][0];
      for (int q = 1; q < 8; q++) if (sh[w][q].valid) bv_take(&b, sh[w][q].p, sh[w][q].len, w);
      cand[(static_cast<size_t>(blockIdx.x) * 2 + w) * BV_MAXC + c] = b;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0 && nc) atomicMax(&out->n_comps, nc);
}

// One CTA: the winners over all CTAs of k_boundary_values, copied out.
__global__ void __launch_bounds__(64) k_boundary_values_finish(const BvCand* cand, uint32_t grid, BvOut* out) {
  const uint32_t nc = out->n_comps;
  const uint32_t t = threadIdx.x;                  // (which, component)
  if (t >= 2 * BV_MAXC) return;
  const int w = t / BV_MAXC; const uint32_t c = t % BV_MAXC;
  if (c >= nc) { out->len[w][c] = 0; return; }
  BvCand b; b.p = nullptr; b.len = 0; b.valid = 0;
  for (uint32_t g = 0; g < grid; g++) {
    const BvCand y = cand[(static_cast<size_t>(g) * 2 + w) * BV_MAXC + c];
    if (y.valid) bv_take(&b, y.p, y.len, w);
  }
  if (!b.valid) { out->len[w][c] = 0; return; }
  if (b.len > BV_MAXLEN) { out->overflow = 1; out->len[w][c] = 0; return; }
  out->len[w][c] = b.len;
  for (uint32_t i = 0; i < b.len; i++) out->val[w][c][i] = b.p[i];
}

}  // namespace ybgpu
