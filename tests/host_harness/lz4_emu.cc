// TEST-ONLY: the LZ4 kernels of yugabyte-db_b200/csrc/lz4_kernels.cuh (the kernel SOURCE, unchanged) on the emulated
// warps of warp_emu.cc, which this file includes whole: its stand-ins, its RunWarp and its entry points
// (we_uncompress_table runs k_snappy_sizes + k_snappy_decode, which dispatch LZ4 blocks to lz4_warp_decode). Built by
// tests/lz4_util.py. Not part of the product.
#include "warp_emu.cc"

extern "C" {

// The engine's LZ4 output pass over a table of `nblocks` assembled blocks (contents + 5-byte trailer back to back at
// raw_off): k_lz4_compress, the prefix sum the engine does with its scan kernels, k_snappy_gather. out must hold
// raw_off[nblocks] bytes; final_off gets nblocks + 1 offsets. Returns the final table length.
uint64_t we_lz4_compress_table(const uint8_t* raw, const uint64_t* raw_off, uint32_t nblocks, uint8_t* out, uint64_t* final_off) {
  using namespace ybgpu;
  InitCrc();
  const uint64_t total = raw_off[nblocks];
  std::vector<uint8_t> rawp(total + 128, 0), comp(total + 128, 0);
  memcpy(rawp.data() + 32, raw, total);
  std::vector<unsigned long long> off(raw_off, raw_off + nblocks + 1), fsize(nblocks + 1, 0);
  std::vector<uint32_t> csize(nblocks, 0);
  SnapCompView V{};
  V.raw = rawp.data() + 32; V.raw_off = off.data(); V.comp = comp.data() + 32; V.csize = csize.data(); V.fsize = fsize.data(); V.nblocks = nblocks;
  RunWarp([&] { k_lz4_compress(V); });
  unsigned long long acc = 0;
  for (uint32_t b = 0; b < nblocks; b++) { const unsigned long long s = fsize[b]; fsize[b] = acc; acc += s; }
  fsize[nblocks] = acc;
  std::vector<uint8_t> outp(acc + 128, 0);
  V.out = outp.data() + 32;
  RunWarp([&] { k_snappy_gather(V); });
  memcpy(out, outp.data() + 32, acc);
  for (uint32_t b = 0; b <= nblocks; b++) final_off[b] = fsize[b];
  return acc;
}

}  // extern "C"
