// TEST-ONLY: the judgement of the output check (yugabyte-db_b200/csrc/dev_logic.cuh verify_interval and friends, what
// k_verify_blocks in verify_kernels.cuh runs one lane per restart interval) on the CPU, block by block and interval by
// interval in the kernel's order: 32 intervals per round, the joins between neighbouring intervals, the join into the next
// block, the per-block entry count and the comparison with the entries that belong in the table. Checksums and
// uncompression are done by the caller (tests/test_verify_cpu.py) and arrive as a per-block verdict. Built and loaded by
// that test; not part of the product.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../yugabyte-db_b200/csrc/dev_logic.cuh"

using namespace ybgpu;

namespace {
struct ExpectKv {
  const uint8_t* keys; const uint64_t* koff; const uint8_t* vals; const uint64_t* voff; uint64_t n;
  bool operator()(uint32_t j, const uint8_t* key, uint32_t klen, const uint8_t* val, uint32_t vlen) const {
    if (j >= n || koff[j + 1] - koff[j] != klen || voff[j + 1] - voff[j] != vlen) return false;
    return memcmp(keys + koff[j], key, klen) == 0 && memcmp(vals + voff[j], val, vlen) == 0;
  }
};
}  // namespace

extern "C" {

// data: the table as BlockIter sees it (blocks uncompressed), block b at off[b] with size[b] bytes of contents.
// pre_kind[b]: VERIFY_CHECKSUM / VERIFY_COMPRESSED when the stored block failed before it could be parsed, else 0.
// block_first (nblocks + 1 entries) + the kv arrays: the entries that belong in the table, or null for a table with
// nothing to compare it with. Returns verify_pack() of the first failure, ~0 when the table is good.
uint64_t vt_verify(const uint8_t* data, const uint64_t* off, const uint32_t* size, const uint8_t* pre_kind, uint32_t nblocks,
                   int key_encoding, uint32_t ri, const uint32_t* block_first, const uint8_t* keys, const uint64_t* koff,
                   const uint8_t* vals, const uint64_t* voff, uint64_t* entries) {
  unsigned long long fail = ~0ull;
  auto note = [&](unsigned long long f) { fail = std::min(fail, f); };
  const bool job = block_first != nullptr;
  const ExpectKv ex{keys, koff, vals, voff, job ? block_first[nblocks] : 0};
  std::vector<std::vector<uint8_t>> bufs(64, std::vector<uint8_t>(VERIFY_MAX_IKEY + 16));
  uint64_t total = 0;
  for (uint32_t b = 0; b < nblocks; b++) {
    if (pre_kind[b]) { note(verify_pack(b, 0, pre_kind[b])); continue; }
    // an exact copy of the block: a read outside it is a read outside the allocation
    std::vector<uint8_t> copy(data + off[b], data + off[b] + size[b]);
    const uint8_t* blk = copy.data();
    uint32_t nres = 0, roff = 0, count = 0;
    if (!verify_block_layout(blk, size[b], &nres, &roff)) { note(verify_pack(b, 0, VERIFY_PARSE)); continue; }
    std::vector<uint8_t> carry; VerifyWalk last{};
    const unsigned long long before = fail;
    fail = ~0ull;                                          // this block's failures; merged below
    for (uint32_t r0 = 0; r0 < nres; r0 += 32) {
      VerifyWalk w[32]; bool have_first[32]; const uint8_t* fkey[32]; uint32_t fklen[32];
      const uint32_t lanes = std::min<uint32_t>(32, nres - r0);
      bool join0 = false;
      for (uint32_t l = 0; l < lanes; l++) {
        const uint32_t r = r0 + l;
        uint32_t p = 0, end = 0;
        const bool ok = verify_interval_bounds(blk, nres, roff, r, &p, &end);
        have_first[l] = ok && verify_restart_key(blk, p, end, key_encoding, &fkey[l], &fklen[l]);
        if (l == 0 && have_first[0] && !carry.empty()) join0 = cmp_internal_keys(carry.data(), static_cast<uint32_t>(carry.size()), fkey[0], fklen[0]) >= 0;
        w[l] = VerifyWalk{};
        if (!ok) { w[l].kind = VERIFY_PARSE; continue; }
        uint8_t* b0 = bufs[2 * l].data(); uint8_t* b1 = bufs[2 * l + 1].data();
        if (job) verify_interval(blk, p, end, key_encoding, b0, b1, VERIFY_MAX_IKEY, block_first[b] + r * ri, ex, &w[l]);
        else verify_interval(blk, p, end, key_encoding, b0, b1, VERIFY_MAX_IKEY, 0u, VerifyNoExpect{}, &w[l]);
      }
      uint32_t base = count;
      for (uint32_t l = 0; l < lanes; l++) {
        const uint32_t r = r0 + l;
        if (w[l].kind != VERIFY_OK) note(verify_pack(b, base + w[l].n, w[l].kind));
        else if (ri && (r + 1 < nres ? w[l].n != ri : w[l].n > ri)) note(verify_pack(b, base, VERIFY_COUNT));
        bool bad = l == 0 && join0;
        if (l > 0 && have_first[l] && w[l - 1].kind == VERIFY_OK && w[l - 1].n > 0 &&
            cmp_internal_keys(w[l - 1].last_key, w[l - 1].last_klen, fkey[l], fklen[l]) >= 0) bad = true;
        if (bad) note(verify_pack(b, base, VERIFY_ORDER));
        base += w[l].n;
      }
      count = base;
      last = w[lanes - 1];
      carry.clear();
      if (last.kind == VERIFY_OK && last.n > 0) carry.assign(last.last_key, last.last_key + last.last_klen);
    }
    if (!carry.empty() && b + 1 < nblocks && !pre_kind[b + 1]) {
      std::vector<uint8_t> ncopy(data + off[b + 1], data + off[b + 1] + size[b + 1]);
      uint32_t nn = 0, nroff = 0, np = 0, nend = 0; const uint8_t* nkey = nullptr; uint32_t nklen = 0;
      if (verify_block_layout(ncopy.data(), size[b + 1], &nn, &nroff) && verify_interval_bounds(ncopy.data(), nn, nroff, 0, &np, &nend) &&
          verify_restart_key(ncopy.data(), np, nend, key_encoding, &nkey, &nklen) &&
          cmp_internal_keys(carry.data(), static_cast<uint32_t>(carry.size()), nkey, nklen) >= 0)
        note(verify_pack(b + 1, 0, VERIFY_ORDER));
    }
    if (job) {
      const uint32_t expect = block_first[b + 1] - block_first[b];
      if (fail == ~0ull && count != expect) note(verify_pack(b, std::min(count, expect), VERIFY_COUNT));
    }
    fail = std::min(fail, before);
    total += count;
  }
  if (entries) *entries = total;
  if (fail == ~0ull && job && total != block_first[nblocks]) fail = verify_pack(nblocks, 0, VERIFY_COUNT);
  return fail;
}

}  // extern "C"
