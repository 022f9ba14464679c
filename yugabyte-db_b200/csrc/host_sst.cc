// host_sst.cc — see host_sst.h.
#include "host_sst.h"
#include "dev_logic.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <stdexcept>
#include <thread>

#if defined(__SSE4_2__)
#include <nmmintrin.h>
#endif

namespace ybgpu {
namespace host {

namespace {

constexpr size_t kTrailer = 5;                                   // table/format.h:208
constexpr size_t kFooterLen = 53;                                // table/format.h:170
constexpr uint64_t kMagic = 0x88e241b785f4cff7ull;               // block_based_table_builder.cc:195

uint32_t g_tab[256];
bool g_tab_ready = [] {
  for (uint32_t i = 0; i < 256; i++) {
    uint32_t c = i;
    for (int j = 0; j < 8; j++) c = (c >> 1) ^ ((c & 1) ? 0x82F63B78u : 0);
    g_tab[i] = c;
  }
  return true;
}();

inline void AppendVarint(std::string* s, uint64_t v) {
  while (v > 0x7f) { s->push_back(static_cast<char>(0x80 | (v & 0x7f))); v >>= 7; }
  s->push_back(static_cast<char>(v));
}
inline size_t VarintLen(uint64_t v) { size_t n = 1; while (v > 0x7f) { v >>= 7; n++; } return n; }
inline void AppendU32(std::string* s, uint32_t v) { s->append(reinterpret_cast<const char*>(&v), 4); }
inline void AppendU64(std::string* s, uint64_t v) { s->append(reinterpret_cast<const char*>(&v), 8); }
inline uint32_t LoadU32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }

bool ReadVarint(const uint8_t** p, const uint8_t* end, uint64_t* out) {
  uint64_t v = 0;
  for (int shift = 0; shift < 64 && *p < end; shift += 7) {
    uint8_t b = *(*p)++;
    v |= static_cast<uint64_t>(b & 0x7f) << shift;
    if (!(b & 0x80)) { *out = v; return true; }
  }
  return false;
}

// Minimal forward reader of a shared-prefix block (index / metaindex / properties blocks always
// use kKeyDeltaEncodingSharedPrefix, table/format.h:46-51, meta_blocks.cc:46-50).
struct BlockCursor {
  const uint8_t* p; const uint8_t* end; std::string key; const uint8_t* val = nullptr; size_t vlen = 0;
  BlockCursor(const uint8_t* data, size_t n) {
    if (n < 4) throw std::runtime_error("bad block contents");
    uint32_t nr = LoadU32(data + n - 4);
    if (static_cast<uint64_t>(nr) * 4 + 4 > n) throw std::runtime_error("bad block contents");
    p = data; end = data + n - 4 - 4 * static_cast<size_t>(nr);
  }
  bool Next() {
    if (p >= end) return false;
    uint64_t shared, non_shared, vl;
    if (!ReadVarint(&p, end, &shared) || !ReadVarint(&p, end, &non_shared) || !ReadVarint(&p, end, &vl) ||
        shared > key.size() || static_cast<uint64_t>(end - p) < non_shared + vl)
      throw std::runtime_error("bad entry in block");
    key.resize(shared);
    key.append(reinterpret_cast<const char*>(p), non_shared);
    val = p + non_shared; vlen = vl;
    p += non_shared + vl;
    return true;
  }
};

// Snappy raw format (the block compression of production tables, docdb_rocksdb_util.cc:184; UncompressBlockContents,
// table/format.cc:441-500): varint32 uncompressed length, then elements — tag & 3 == 0: literal of (tag >> 2) + 1 bytes
// (60..63: the length - 1 follows in 1..4 little-endian bytes); 1: copy, length 4 + ((tag >> 2) & 7), offset = (tag >> 5)
// << 8 | next byte; 2 / 3: copy, length (tag >> 2) + 1, offset in the next 2 / 4 bytes. Copies may overlap their output.
// Index blocks of the metadata file go through WriteBlock like data blocks (block_based_table_builder.cc:586,790,823,869)
// and so are stored compressed in production files; data blocks are uncompressed on the GPU (snappy_kernels.cuh).
void SnappyUncompress(const uint8_t* in, size_t n, std::string* out) {
  const uint8_t* p = in; const uint8_t* end = in + n;
  uint64_t ulen = 0;
  if (!ReadVarint(&p, end, &ulen) || ulen > (1ull << 32)) throw std::runtime_error("bad compressed block (length)");
  out->clear();
  out->reserve(ulen);
  while (p < end) {
    const uint32_t tag = *p++;
    uint64_t len, off = 0;
    if ((tag & 3) == 0) {
      len = (tag >> 2) + 1;
      if (len > 60) {
        const uint32_t nb = static_cast<uint32_t>(len - 60);
        if (static_cast<size_t>(end - p) < nb) throw std::runtime_error("bad compressed block (literal length)");
        len = 0;
        for (uint32_t i = 0; i < nb; i++) len |= static_cast<uint64_t>(p[i]) << (8 * i);
        len += 1; p += nb;
      }
      if (static_cast<uint64_t>(end - p) < len || out->size() + len > ulen) throw std::runtime_error("bad compressed block (literal)");
      out->append(reinterpret_cast<const char*>(p), len);
      p += len;
      continue;
    }
    if ((tag & 3) == 1) {
      if (p >= end) throw std::runtime_error("bad compressed block (copy)");
      len = 4 + ((tag >> 2) & 7); off = (static_cast<uint64_t>(tag >> 5) << 8) | *p++;
    } else {
      const uint32_t nb = (tag & 3) == 2 ? 2 : 4;
      if (static_cast<size_t>(end - p) < nb) throw std::runtime_error("bad compressed block (copy)");
      len = (tag >> 2) + 1;
      for (uint32_t i = 0; i < nb; i++) off |= static_cast<uint64_t>(p[i]) << (8 * i);
      p += nb;
    }
    if (off == 0 || off > out->size() || out->size() + len > ulen) throw std::runtime_error("bad compressed block (copy offset)");
    const size_t from = out->size() - off;
    for (uint64_t i = 0; i < len; i++) out->push_back((*out)[from + i]);
  }
  if (out->size() != ulen) throw std::runtime_error("bad compressed block (short)");
}

// The writer's side (block_based_table_builder.cc:115-131 CompressBlock with kSnappyCompression). Same element choice
// as the GPU kernel (snappy_kernels.cuh k_snappy_compress), so that the index blocks written here and the data blocks
// written there come from one encoder: 64 KB fragments; per fragment a table of 2^12 fragment-relative positions keyed
// by a multiplicative hash of the next four bytes; every visited position replaces its slot's occupant and tries it as
// the match candidate; a match is extended as far as it goes and cut into copy elements of at most 64 bytes (none
// shorter than four); positions inside a match are not visited.
void SnappyCompress(const uint8_t* raw, size_t total, std::string* out) {
  out->clear();
  AppendVarint(out, total);
  uint16_t table[1 << 12];
  for (size_t fs = 0; fs < total; fs += 65536) {
    const uint8_t* f = raw + fs;
    const size_t m = std::min<size_t>(65536, total - fs);
    memset(table, 0, sizeof(table));
    size_t lit = 0, i = 0;
    auto literal = [&](size_t to) {
      if (to == lit) return;
      const size_t l1 = to - lit - 1;
      if (l1 < 60) { out->push_back(static_cast<char>(l1 << 2)); }
      else if (l1 < 256) { out->push_back(static_cast<char>(60 << 2)); out->push_back(static_cast<char>(l1)); }
      else { out->push_back(static_cast<char>(61 << 2)); out->push_back(static_cast<char>(l1 & 0xff)); out->push_back(static_cast<char>(l1 >> 8)); }
      out->append(reinterpret_cast<const char*>(f + lit), to - lit);
    };
    while (i + 4 <= m) {
      uint32_t w; memcpy(&w, f + i, 4);
      uint16_t& slot = table[(w * 0x1e35a7bdu) >> 20];
      const size_t cand = slot;
      slot = static_cast<uint16_t>(i);
      if (cand >= i || memcmp(f + cand, f + i, 4) != 0) { i++; continue; }
      size_t len = 4;
      while (i + len < m && f[cand + len] == f[i + len]) len++;
      literal(i);
      const uint32_t off = static_cast<uint32_t>(i - cand);
      for (size_t left = len; left;) {
        size_t l = std::min<size_t>(left, 64);
        if (left > l && left - l < 4) l = left - 4;
        if (l <= 11 && off < 2048) {
          out->push_back(static_cast<char>(1 | ((l - 4) << 2) | ((off >> 8) << 5))); out->push_back(static_cast<char>(off & 0xff));
        } else {
          out->push_back(static_cast<char>(2 | ((l - 1) << 2))); out->push_back(static_cast<char>(off & 0xff)); out->push_back(static_cast<char>(off >> 8));
        }
        left -= l;
      }
      i += len; lit = i;
    }
    literal(m);
  }
}

// kLZ4Compression / kLZ4HCCompression with compress_format_version 2 (util/compression.h LZ4_Uncompress): varint32
// uncompressed length, then one raw LZ4 block — sequences of a token (literal length << 4 | match length - 4; a nibble
// of 15 continues in bytes that add their value, 255 = more follow), literals, a 2-byte offset, match-length bytes.
// Rejects what LZ4_decompress_safe rejects with the announced length as the capacity: the last sequence is literals
// only, the last 5 output bytes are literals, no match starts within the last 12; and an output of any other length.
void Lz4Uncompress(const uint8_t* in, size_t n, std::string* out) {
  const uint8_t* p = in; const uint8_t* end = in + n;
  uint64_t ulen = 0;
  if (!ReadVarint(&p, end, &ulen) || ulen > (1ull << 32)) throw std::runtime_error("bad compressed block (length)");
  out->clear();
  out->reserve(ulen);
  auto ext = [&](uint64_t* len) {
    uint32_t b;
    do {
      if (p >= end) throw std::runtime_error("bad compressed block (length byte)");
      b = *p++;
      *len += b;
      if (*len > ulen) throw std::runtime_error("bad compressed block (long)");
    } while (b == 255);
  };
  for (;;) {
    if (p >= end) throw std::runtime_error("bad compressed block (token)");
    const uint32_t token = *p++;
    uint64_t lit = token >> 4;
    if (lit == 15) ext(&lit);
    if (static_cast<uint64_t>(end - p) < lit || out->size() + lit > ulen) throw std::runtime_error("bad compressed block (literal)");
    out->append(reinterpret_cast<const char*>(p), lit);
    p += lit;
    if (p == end) break;                                   // the last sequence: literals only
    if (out->size() + 12 > ulen || end - p < 2) throw std::runtime_error("bad compressed block (match position)");
    const uint64_t off = p[0] | (static_cast<uint64_t>(p[1]) << 8);
    p += 2;
    uint64_t len = token & 15;
    if (len == 15) ext(&len);
    len += 4;
    if (off == 0 || off > out->size() || out->size() + len + 5 > ulen) throw std::runtime_error("bad compressed block (match)");
    const size_t from = out->size() - off;
    for (uint64_t i = 0; i < len; i++) out->push_back((*out)[from + i]);
  }
  if (out->size() != ulen) throw std::runtime_error("bad compressed block (short)");
}

// The writer's side, kLZ4Compression: the one LZ4 encoder of the engine. The GPU kernel (lz4_kernels.cuh
// k_lz4_compress) emits the same sequences, so the index blocks written here and the data blocks written there come from
// one encoder (and the test suite's reference, tests/lz4_util.py, restates it). The search is SnappyCompress's:
//   * 64 KB fragments; per fragment a table of 2^12 u16 fragment-relative positions, zeroed at the fragment's start;
//   * the hash (w * 0x1e35a7bd) >> 20 of the four bytes w at a position; every visited position takes its slot and
//     tries the slot's previous occupant as the match candidate; greedy, no skipping; positions inside a match are not
//     visited; a match never reaches back across the fragment's start, so an offset is at most 65535.
// What LZ4 adds:
//   * literal runs span fragments: the pending literal starts at a block-absolute position, and a sequence's literals
//     are emitted with its match, as one token;
//   * end-of-block limits: a position p (block-absolute) is tried only while p <= n - 12 and p + 4 <= the fragment's
//     end; a match is extended no further than min(fragment end, n - 5); the block ends with one literals-only sequence,
//     empty only when the block is;
//   * the varint32 preamble comes first. The GPU kernel abandons a block as soon as its output reaches n - n/8 (the
//     GoodCompressionRatio bound); this function writes the whole stream and AppendBlockTo applies the same bound, which
//     comes to the same decision since the stream only grows.
// It is NOT liblz4's encoder: the compressed bytes are this encoder's; the format is liblz4's (tests decode every stream
// with liblz4 and pyarrow's lz4_raw).
void Lz4Compress(const uint8_t* raw, size_t n, std::string* out) {
  out->clear();
  AppendVarint(out, n);
  auto put_len = [&](size_t v) {
    for (v -= 15; v >= 255; v -= 255) out->push_back(static_cast<char>(255));
    out->push_back(static_cast<char>(v));
  };
  size_t lit = 0;
  auto sequence = [&](size_t to, size_t mlen, uint32_t off) {
    const size_t L = to - lit, M = mlen ? mlen - 4 : 0;
    out->push_back(static_cast<char>((std::min<size_t>(L, 15) << 4) | std::min<size_t>(M, 15)));
    if (L >= 15) put_len(L);
    out->append(reinterpret_cast<const char*>(raw + lit), L);
    if (!mlen) return;
    out->push_back(static_cast<char>(off & 0xff)); out->push_back(static_cast<char>(off >> 8));
    if (M >= 15) put_len(M);
  };
  uint16_t table[1 << 12];
  for (size_t fs = 0; fs < n; fs += 65536) {
    const uint8_t* f = raw + fs;
    const size_t m = std::min<size_t>(65536, n - fs);
    const size_t smax = n - fs > 8 ? std::min<size_t>(m, n - fs - 8) : 0;
    const size_t emax = n - fs > 5 ? std::min<size_t>(m, n - fs - 5) : 0;
    memset(table, 0, sizeof(table));
    size_t i = 0;
    while (i + 4 <= smax) {
      uint32_t w; memcpy(&w, f + i, 4);
      uint16_t& slot = table[(w * 0x1e35a7bdu) >> 20];
      const size_t cand = slot;
      slot = static_cast<uint16_t>(i);
      if (cand >= i || memcmp(f + cand, f + i, 4) != 0) { i++; continue; }
      size_t len = 4;
      while (i + len < emax && f[cand + len] == f[i + len]) len++;
      sequence(fs + i, len, static_cast<uint32_t>(i - cand));
      i += len; lit = fs + i;
    }
  }
  sequence(n, 0, 0);
}

// A block of the metadata file, uncompressed if it is stored compressed.
struct LoadedBlock {
  const uint8_t* data = nullptr; size_t size = 0;
  std::string scratch;
};
void LoadBlock(const uint8_t* file, uint64_t len, const Handle& h, LoadedBlock* b) {
  if (h.offset + h.size + kTrailer > len) throw std::runtime_error("block handle outside file");
  const uint8_t type = file[h.offset + h.size];
  if (type == 0) { b->data = file + h.offset; b->size = h.size; return; }
  if (!UncompressStoredBlock(type, file + h.offset, h.size, &b->scratch))
    throw std::runtime_error("metadata block: malformed stream or unsupported codec " + std::to_string(type) + " (Snappy and LZ4 are read)");
  b->data = reinterpret_cast<const uint8_t*>(b->scratch.data()); b->size = b->scratch.size();
}
const uint8_t* BlockAt(const uint8_t* file, uint64_t len, const Handle& h) {
  if (h.offset + h.size + kTrailer > len) throw std::runtime_error("block handle outside file");
  if (file[h.offset + h.size] != 0) throw std::runtime_error("compressed meta block not supported");
  return file + h.offset;
}

Handle ReadHandle(const uint8_t** p, const uint8_t* end) {
  Handle h;
  if (!ReadVarint(p, end, &h.offset) || !ReadVarint(p, end, &h.size)) throw std::runtime_error("bad block handle");
  return h;
}

}  // namespace

bool UncompressStoredBlock(uint8_t type, const uint8_t* stored, size_t n, std::string* out) {
  try {
    if (type == 1) { SnappyUncompress(stored, n, out); return true; }
    if (type == 4 || type == 5) { Lz4Uncompress(stored, n, out); return true; }   // LZ4HC writes the same stream format
    return false;
  } catch (const std::exception&) { return false; }
}

uint32_t Crc32c(const uint8_t* p, size_t n, uint32_t init) {
  uint32_t c = ~init;
#if defined(__SSE4_2__)
  uint64_t c64 = c;
  for (; n >= 8; n -= 8, p += 8) { uint64_t v; memcpy(&v, p, 8); c64 = _mm_crc32_u64(c64, v); }
  c = static_cast<uint32_t>(c64);
  for (; n; n--, p++) c = _mm_crc32_u8(c, *p);
#else
  for (; n; n--, p++) c = g_tab[(c ^ *p) & 0xff] ^ (c >> 8);
#endif
  return ~c;
}

std::string ParseSplitSstMeta(const uint8_t* meta, uint64_t len, SstMeta* out) {
  try {
    if (len < kFooterLen) return "file is too short to be an sstable";
    const uint8_t* f = meta + len - kFooterLen;
    uint64_t magic = static_cast<uint64_t>(LoadU32(f + kFooterLen - 8)) | (static_cast<uint64_t>(LoadU32(f + kFooterLen - 4)) << 32);
    if (magic != kMagic) return "bad table magic number";
    const uint8_t* p = f + 1;
    Handle metaindex = ReadHandle(&p, f + 41);
    Handle index = ReadHandle(&p, f + 41);
    BlockCursor mi(BlockAt(meta, len, metaindex), metaindex.size);
    while (mi.Next()) {
      if (mi.key.compare(0, 16, "fixedsizefilter.") == 0) {
        out->filter_policy_name = mi.key.substr(16);
        const uint8_t* vp = mi.val;
        Handle fh = ReadHandle(&vp, mi.val + mi.vlen);
        LoadedBlock fib;
        LoadBlock(meta, len, fh, &fib);                  // the filter index is an index block: compressed in production files
        BlockCursor fi(fib.data, fib.size);
        while (fi.Next()) {
          const uint8_t* hp = fi.val;
          Handle bh = ReadHandle(&hp, fi.val + fi.vlen);
          BlockAt(meta, len, bh);
          out->filter_blocks.push_back(bh);
          out->filter_index_keys.push_back(fi.key);
        }
      }
      if (mi.key == "rocksdb.properties") {
        const uint8_t* vp = mi.val;
        Handle ph = ReadHandle(&vp, mi.val + mi.vlen);
        BlockCursor props(BlockAt(meta, len, ph), ph.size);
        while (props.Next()) out->properties[props.key] = std::string(reinterpret_cast<const char*>(props.val), props.vlen);
      }
    }
    auto e = out->properties.find("rocksdb.block.based.table.data.block.key.value.encoding.format");
    out->key_encoding = (e == out->properties.end() || e->second.empty()) ? 1 : static_cast<uint8_t>(e->second[0]);
    auto l = out->properties.find("rocksdb.block.based.table.index.num.levels");
    out->index_levels = (l == out->properties.end() || l->second.size() < 4)
                            ? 1 : static_cast<int>(LoadU32(reinterpret_cast<const uint8_t*>(l->second.data())));
    std::vector<Handle> level{index};
    for (int lv = 0; lv < out->index_levels; lv++) {
      std::vector<Handle> next;
      const bool last_level = lv + 1 == out->index_levels;
      for (const Handle& h : level) {
        LoadedBlock ib;
        LoadBlock(meta, len, h, &ib);
        BlockCursor c(ib.data, ib.size);
        while (c.Next()) {
          const uint8_t* vp = c.val; next.push_back(ReadHandle(&vp, c.val + c.vlen));
          if (last_level) out->separators.push_back(c.key);
        }
      }
      level.swap(next);
    }
    out->data_blocks.swap(level);
    return std::string();
  } catch (const std::exception& ex) {
    return ex.what();
  }
}

// ---------------------------------------------------------------------------------------------
BlockEncoder::BlockEncoder(int restart_interval, int key_encoding) : interval_(restart_interval), encoding_(key_encoding) {
  restarts_.push_back(0);
}

void BlockEncoder::Reset() {
  body_.clear(); last_key_.clear(); restarts_.assign(1, 0); in_interval_ = 0; finished_ = false;
}

size_t BlockEncoder::SizeAfter(size_t klen, size_t vlen) const {   // block_builder.cc:94-108
  size_t e = SizeEstimate() + klen + vlen;
  if (in_interval_ >= interval_) e += 4;
  return e + 4 + VarintLen(klen) + VarintLen(vlen);
}

void BlockEncoder::Add(const uint8_t* key, size_t klen, const uint8_t* val, size_t vlen) {
  size_t shared = 0;
  if (in_interval_ >= interval_) {
    restarts_.push_back(static_cast<uint32_t>(body_.size()));
    in_interval_ = 0;
  } else {
    const size_t lim = std::min(last_key_.size(), klen);
    const uint8_t* prev = reinterpret_cast<const uint8_t*>(last_key_.data());
    while (shared < lim && prev[shared] == key[shared]) shared++;
  }
  if (encoding_ == 2 && klen >= 8) {
    // kKeyDeltaEncodingThreeSharedParts (block_builder.cc:265-333): same planner as the GPU encoder
    const bool restart = in_interval_ == 0;
    auto ref = [](const uint8_t* k, size_t n) {
      uint64_t suf = 0;
      for (int i = 7; i >= 0; i--) suf = (suf << 8) | k[n - 8 + i];
      return IKeyRef{k, static_cast<uint32_t>(n - 8), suf};
    };
    const IKeyRef kk = ref(key, klen);
    const IKeyRef pk = (restart || last_key_.size() < 8) ? IKeyRef{nullptr, 0, 0}
                                                         : ref(reinterpret_cast<const uint8_t*>(last_key_.data()), last_key_.size());
    TspPlan pl;
    tsp_plan(pk, kk, static_cast<uint32_t>(vlen), restart, static_cast<uint32_t>(shared), &pl);
    body_.append(reinterpret_cast<const char*>(pl.hdr), pl.hdr_len);
    body_.append(reinterpret_cast<const char*>(key + pl.shared), pl.ns1);
    body_.append(reinterpret_cast<const char*>(key + klen - pl.last_reuse - pl.ns2), pl.ns2);
  } else {
    AppendVarint(&body_, shared);
    AppendVarint(&body_, klen - shared);
    AppendVarint(&body_, vlen);
    body_.append(reinterpret_cast<const char*>(key + shared), klen - shared);
  }
  body_.append(reinterpret_cast<const char*>(val), vlen);
  last_key_.assign(reinterpret_cast<const char*>(key), klen);
  in_interval_++;
}

const std::string& BlockEncoder::Finish() {
  for (uint32_t r : restarts_) AppendU32(&body_, r);
  AppendU32(&body_, static_cast<uint32_t>(restarts_.size()));
  finished_ = true;
  return body_;
}

// ---------------------------------------------------------------------------------------------
// Separator shortening (util/comparator.cc:53-93, db/dbformat.cc:139-172).
static void ShortenUserSeparator(std::string* start, const uint8_t* limit, size_t llen) {
  const size_t lim = std::min(start->size(), llen);
  size_t d = 0;
  while (d < lim && static_cast<uint8_t>((*start)[d]) == limit[d]) d++;
  if (d >= lim) return;
  const uint8_t a = static_cast<uint8_t>((*start)[d]), b = limit[d];
  if (a > b) return;
  if (d == llen - 1 && a + 1 == b) {
    ++d;
    while (d < start->size() && static_cast<uint8_t>((*start)[d]) == 0xff) ++d;
    if (d == start->size()) return;
  }
  (*start)[d] = static_cast<char>(static_cast<uint8_t>((*start)[d]) + 1);
  start->resize(d + 1);
}

static int CompareBytes(const std::string& a, const std::string& b) {
  const size_t m = std::min(a.size(), b.size());
  int r = m ? memcmp(a.data(), b.data(), m) : 0;
  if (r == 0) r = a.size() < b.size() ? -1 : (a.size() > b.size() ? 1 : 0);
  return r;
}

static const uint64_t kSeekSuffix = (((1ull << 56) - 1) << 8) | 7;   // kMaxSequenceNumber, kValueTypeForSeek

static void InternalSeparator(std::string* key, const uint8_t* limit, size_t llen) {
  std::string user(key->data(), key->size() - 8), tmp = user;
  ShortenUserSeparator(&tmp, limit, llen - 8);
  if (tmp.size() < user.size() && CompareBytes(user, tmp) < 0) { AppendU64(&tmp, kSeekSuffix); key->swap(tmp); }
}

static void InternalSuccessor(std::string* key) {
  std::string user(key->data(), key->size() - 8), tmp = user;
  for (size_t i = 0; i < tmp.size(); i++) {
    if (static_cast<uint8_t>(tmp[i]) != 0xff) { tmp[i] = static_cast<char>(static_cast<uint8_t>(tmp[i]) + 1); tmp.resize(i + 1); break; }
  }
  if (tmp.size() < user.size() && CompareBytes(user, tmp) < 0) { AppendU64(&tmp, kSeekSuffix); key->swap(tmp); }
}

// Multi-level index. Level L collects one entry per finished block of level L-1 (level 0: per
// data block). A level's block is cut by the size policy evaluated after each added entry
// (index_builder.cc:170-196); the finished block's own entry is added to level L+1 on the next
// flush round, after which a full level-L+1 block is written BEFORE the pending level-L block
// (index_builder.cc:228-249). The explicit per-level state below replays exactly that order.
class IndexWriter {
 public:
  explicit IndexWriter(const TableOptions& o) : o_(o) { levels_.emplace_back(new Level(o)); }

  void AddDataBlock(std::string* last_key, const uint8_t* next_key, size_t next_len, bool has_next, const Handle& h) {
    if (!has_next) InternalSuccessor(last_key); else InternalSeparator(last_key, next_key, next_len);
    AddEntry(0, *last_key, has_next ? std::string(reinterpret_cast<const char*>(next_key), next_len) : std::string(), has_next, h);
  }
  void AddRaw(const std::string& index_key, bool has_next, const Handle& h) { AddEntry(0, index_key, std::string(), has_next, h); }
  bool ShouldFlush(size_t lv = 0) const {
    const Level& L = *levels_[lv];
    return L.ready.on || (L.to_parent.on && !L.to_parent.has_next) || (lv + 1 < levels_.size() && ShouldFlush(lv + 1));
  }
  // One flush step: true => *contents must be written, its handle reported via the next call.
  bool FlushNext(std::string* contents, const Handle& last_written, bool last_written_set, size_t lv = 0) {
    Level& L = *levels_[lv];
    if (L.parent_just_flushed) { L.parent_last = last_written; L.parent_last_set = last_written_set; L.parent_just_flushed = false; }
    if (L.flushing) {
      if (L.to_parent.on) {
        AddEntry(lv + 1, L.to_parent.last_key, L.to_parent.next_first, L.to_parent.has_next, last_written);
        L.to_parent.on = false;
      }
      if (lv + 1 < levels_.size() && ShouldFlush(lv + 1)) {
        bool r = FlushNext(contents, L.parent_last, L.parent_last_set, lv + 1);
        L.parent_just_flushed = true;
        return r;
      }
    }
    L.flushing = true;
    if (L.ready.on) {
      Emit(&L, contents);
      if (lv + 1 == levels_.size() && L.ready.has_next) levels_.emplace_back(new Level(o_));
      if (lv + 1 < levels_.size()) L.to_parent = L.ready;
      L.ready.on = false;
      return true;
    }
    if (!last_written_set) { Emit(&L, contents); return true; }   // empty table: empty index block
    return false;
  }
  size_t EstimatedSize() const {
    size_t s = 0;
    for (auto& l : levels_) s += l->bytes;
    return s - kTrailer;
  }
  int NumLevels() const { return static_cast<int>(levels_.size()); }

 private:
  struct Pending { bool on = false; std::string last_key, next_first; bool has_next = false; };
  struct Level {
    explicit Level(const TableOptions& o) : enc(o.index_block_restart_interval, 1) {}
    BlockEncoder enc;
    Pending ready, to_parent;
    Handle parent_last; bool parent_last_set = false, parent_just_flushed = false, flushing = false;
    size_t bytes = 0;
  };
  void AddEntry(size_t lv, const std::string& key, const std::string& next_first, bool has_next, const Handle& h) {
    while (lv >= levels_.size()) levels_.emplace_back(new Level(o_));
    Level& L = *levels_[lv];
    std::string enc;
    AppendVarint(&enc, h.offset); AppendVarint(&enc, h.size);
    L.enc.Add(reinterpret_cast<const uint8_t*>(key.data()), key.size(), reinterpret_cast<const uint8_t*>(enc.data()), enc.size());
    const size_t cur = L.enc.SizeEstimate();
    const bool almost = L.enc.SizeAfter(key.size(), enc.size()) > o_.index_block_size && o_.block_size_deviation > 0 &&
                        cur * 100 > static_cast<size_t>(o_.index_block_size) * (100 - o_.block_size_deviation);
    const bool cut = (cur >= o_.index_block_size || almost) && L.enc.NumKeysForPolicy() >= o_.min_keys_per_index_block;
    if (cut || !has_next) { L.ready.on = true; L.ready.last_key = key; L.ready.has_next = has_next; L.ready.next_first = next_first; }
  }
  void Emit(Level* L, std::string* contents) {
    *contents = L->enc.Finish();
    L->enc.Reset();
    L->bytes += contents->size() + kTrailer;
  }
  TableOptions o_;
  std::vector<std::unique_ptr<Level>> levels_;
};

// ---------------------------------------------------------------------------------------------
// WriteBlock + WriteRawBlock (block_based_table_builder.cc:630-707): `compression` 1 / 4 = stored Snappy- / LZ4-compressed
// when that saves at least 12.5 % (GoodCompressionRatio :109-112); blocks of 2 GB and more are never compressed (:642).
static void AppendBlockTo(const std::string& raw, std::string* file, Handle* h, int compression = 0) {
  std::string packed;
  uint8_t type = 0;
  if ((compression == 1 || compression == 4) && raw.size() < 0x7fffffffull) {
    if (compression == 1) SnappyCompress(reinterpret_cast<const uint8_t*>(raw.data()), raw.size(), &packed);
    else Lz4Compress(reinterpret_cast<const uint8_t*>(raw.data()), raw.size(), &packed);
    if (packed.size() < raw.size() - raw.size() / 8u) type = static_cast<uint8_t>(compression);
  }
  const std::string& c = type ? packed : raw;
  h->offset = file->size(); h->size = c.size();
  file->append(c);
  uint32_t crc = Crc32c(&type, 1, Crc32c(reinterpret_cast<const uint8_t*>(c.data()), c.size()));
  file->push_back(static_cast<char>(type));
  AppendU32(file, Crc32cMask(crc));
}

FilterGeometry ComputeFilterGeometry(uint32_t block_bytes) {
  // same double arithmetic, in the same order, as FixedSizeFilterBitsBuilder's ctor (bloom.cc:389-415)
  FilterGeometry g;
  const double kLog2 = std::log(2.0), error_rate = 0.01;
  const size_t total_bits_in = static_cast<size_t>(block_bytes) * 8;
  size_t num_lines = (total_bits_in + 64 * 8 - 1) / (64 * 8);
  if (num_lines % 2 == 0) { if (num_lines * 64 < 4096) num_lines++; else num_lines--; }
  const size_t total_bits = num_lines * 64 * 8;
  const double minus_log_error_rate = -std::log(error_rate);
  size_t num_probes = static_cast<size_t>(minus_log_error_rate / kLog2);
  num_probes = std::max<size_t>(num_probes, 1);
  num_probes = std::min<size_t>(num_probes, 255);
  const double max_keys = total_bits * kLog2 * kLog2 / minus_log_error_rate;
  g.num_lines = static_cast<uint32_t>(num_lines); g.num_probes = static_cast<uint32_t>(num_probes);
  g.max_keys = static_cast<uint32_t>(static_cast<size_t>(max_keys));
  g.filter_bytes = static_cast<uint32_t>(total_bits / 8 + 5);
  return g;
}

// util/comparator.cc:53-93 BytewiseComparator::FindShortSuccessor
static void ShortSuccessor(std::string* key) {
  for (size_t i = 0; i < key->size(); i++) {
    const uint8_t b = static_cast<uint8_t>((*key)[i]);
    if (b != 0xff) { (*key)[i] = static_cast<char>(b + 1); key->resize(i + 1); return; }
  }
}

MetaFileWriter::MetaFileWriter(const TableOptions& o) : o_(o), index_(new IndexWriter(o)) {
  if (o.filter_policy) filter_index_.reset(new BlockEncoder(o.index_block_restart_interval, 1));
}
MetaFileWriter::~MetaFileWriter() {}
// Index blocks and the filter index go through WriteBlock (compressible); filter blocks, properties and the
// metaindex through WriteRawBlock with kNoCompression (block_based_table_builder.cc:586,600,790,823,849,864,869).
void MetaFileWriter::AppendBlock(const std::string& c, Handle* h, bool compressible) {
  AppendBlockTo(c, &meta_, h, compressible ? o_.compression : 0);
}

void MetaFileWriter::AddDataBlock(std::string* last_key, const uint8_t* next_key, size_t next_len, bool has_next, const Handle& h) {
  index_->AddDataBlock(last_key, next_key, next_len, has_next, h);
  while (index_->ShouldFlush()) {
    std::string contents;
    if (!index_->FlushNext(&contents, last_index_, last_index_set_)) throw std::runtime_error("index flush failed");
    AppendBlock(contents, &last_index_, true);
    last_index_set_ = true;
    num_index_blocks_++;
  }
}

void MetaFileWriter::AddFilterBlock(const uint8_t* contents, size_t len, std::string* last_filter_key, const uint8_t* next_key, size_t next_len,
                                    bool has_next) {
  Handle h;
  AppendBlock(std::string(reinterpret_cast<const char*>(contents), len), &h);
  filter_size_ += len + kTrailer;
  num_filter_blocks_++;
  // ShortenedIndexBuilder::AddIndexEntry with BytewiseComparator (index_builder.cc:60-86)
  if (has_next) ShortenUserSeparator(last_filter_key, next_key, next_len); else ShortSuccessor(last_filter_key);
  std::string enc; AppendVarint(&enc, h.offset); AppendVarint(&enc, h.size);
  filter_index_->Add(reinterpret_cast<const uint8_t*>(last_filter_key->data()), last_filter_key->size(),
                     reinterpret_cast<const uint8_t*>(enc.data()), enc.size());
}

void MetaFileWriter::AddDataBlockRaw(const std::string& index_key, bool has_next, const Handle& h) {
  index_->AddRaw(index_key, has_next, h);
  while (index_->ShouldFlush()) {
    std::string contents;
    if (!index_->FlushNext(&contents, last_index_, last_index_set_)) throw std::runtime_error("index flush failed");
    AppendBlock(contents, &last_index_, true);
    last_index_set_ = true;
    num_index_blocks_++;
  }
}

void MetaFileWriter::AddFilterBlockRaw(const uint8_t* contents, size_t len, const std::string& filter_index_key) {
  Handle h;
  AppendBlock(std::string(reinterpret_cast<const char*>(contents), len), &h);   // + trailer (type byte, masked CRC32C)
  filter_size_ += len + kTrailer;
  num_filter_blocks_++;
  std::string enc; AppendVarint(&enc, h.offset); AppendVarint(&enc, h.size);
  filter_index_->Add(reinterpret_cast<const uint8_t*>(filter_index_key.data()), filter_index_key.size(),
                     reinterpret_cast<const uint8_t*>(enc.data()), enc.size());
}

void MetaFileWriter::Finish(const MetaProps& mp) {
  std::string top;
  const bool have_top = index_->FlushNext(&top, last_index_, last_index_set_);
  if (have_top) num_index_blocks_++;
  std::map<std::string, std::string> props;
  auto num = [&](const char* name, uint64_t v) { std::string s; AppendVarint(&s, v); props[name] = s; };
  num("rocksdb.raw.key.size", mp.raw_key_size);
  num("rocksdb.raw.value.size", mp.raw_value_size);
  num("rocksdb.data.size", mp.data_size);
  num("rocksdb.data.index.size", index_->EstimatedSize() + kTrailer);
  num("rocksdb.filter.index.size", 0);
  num("rocksdb.num.entries", mp.num_entries);
  num("rocksdb.num.data.blocks", mp.num_data_blocks);
  num("rocksdb.num.filter.blocks", 0);
  num("rocksdb.num.data.index.blocks", num_index_blocks_);
  num("rocksdb.filter.size", 0);
  num("rocksdb.format.version", 0);
  num("rocksdb.fixed.key.length", 0);
  num("rocksdb.deleted.keys", mp.deleted_keys);
  { std::string v; AppendU32(&v, 2); props["rocksdb.block.based.table.index.type"] = v; }   // kMultiLevelBinarySearch
  props["rocksdb.block.based.table.whole.key.filtering"] = "1";
  props["rocksdb.block.based.table.prefix.filtering"] = "0";
  { std::string v; AppendU32(&v, static_cast<uint32_t>(index_->NumLevels())); props["rocksdb.block.based.table.index.num.levels"] = v; }
  props["rocksdb.block.based.table.data.block.key.value.encoding.format"] = std::string(1, static_cast<char>(o_.key_encoding));
  Handle filter_index_handle;
  if (filter_index_) {
    // filter index block, then its metaindex entry (block_based_table_builder.cc:795-830)
    const std::string& fi = filter_index_->Finish();
    AppendBlock(fi, &filter_index_handle, true);
    num("rocksdb.filter.index.size", filter_index_->SizeEstimate() + kTrailer);
    num("rocksdb.num.filter.blocks", num_filter_blocks_);
    num("rocksdb.filter.size", filter_size_);
    props["rocksdb.filter.policy"] = "DocKeyV3Filter";
  }
  BlockEncoder pb(1, 1);
  for (auto& kv : props)
    pb.Add(reinterpret_cast<const uint8_t*>(kv.first.data()), kv.first.size(), reinterpret_cast<const uint8_t*>(kv.second.data()), kv.second.size());
  Handle ph;
  AppendBlock(pb.Finish(), &ph);
  BlockEncoder mb(1, 1);
  if (filter_index_) {   // MetaIndexBuilder sorts its keys: "fixedsizefilter." < "rocksdb." (meta_blocks.cc:71-83)
    std::string k = "fixedsizefilter.DocKeyV3Filter", v; AppendVarint(&v, filter_index_handle.offset); AppendVarint(&v, filter_index_handle.size);
    mb.Add(reinterpret_cast<const uint8_t*>(k.data()), k.size(), reinterpret_cast<const uint8_t*>(v.data()), v.size());
  }
  { std::string k = "rocksdb.properties", v; AppendVarint(&v, ph.offset); AppendVarint(&v, ph.size);
    mb.Add(reinterpret_cast<const uint8_t*>(k.data()), k.size(), reinterpret_cast<const uint8_t*>(v.data()), v.size()); }
  Handle mh;
  AppendBlock(mb.Finish(), &mh);
  if (have_top) { AppendBlock(top, &last_index_, true); last_index_set_ = true; }
  std::string f;
  f.push_back(1);   // kCRC32c
  AppendVarint(&f, mh.offset); AppendVarint(&f, mh.size);
  AppendVarint(&f, last_index_.offset); AppendVarint(&f, last_index_.size);
  f.resize(kFooterLen - 12);
  AppendU32(&f, 2);
  AppendU32(&f, static_cast<uint32_t>(kMagic & 0xffffffffu));
  AppendU32(&f, static_cast<uint32_t>(kMagic >> 32));
  meta_.append(f);
}

// ---------------------------------------------------------------------------------------------
SplitSstWriter::SplitSstWriter(const TableOptions& o)
    : o_(o), block_(o.block_restart_interval, o.key_encoding), metaw_(o) {
  if (o.key_encoding != 1 && o.key_encoding != 2) throw std::runtime_error("host writer: unknown key-value encoding format");
  if (o.filter_policy) { fg_ = ComputeFilterGeometry(o.filter_block_size); filter_bits_.assign(fg_.filter_bytes, '\0'); }
}
SplitSstWriter::~SplitSstWriter() {}

void SplitSstWriter::Add(const uint8_t* key, size_t klen, const uint8_t* val, size_t vlen) {
  // FlushBlockBySizePolicy::Update (flush_block_policy.cc:45-76), min_keys_per_block = 1
  if (!block_.empty()) {
    const size_t cur = block_.SizeEstimate();
    const bool almost = block_.SizeAfter(klen, vlen) > o_.block_size && o_.block_size_deviation > 0 &&
                        cur * 100 > static_cast<size_t>(o_.block_size) * (100 - o_.block_size_deviation);
    if ((cur >= o_.block_size || almost) && block_.NumKeysForPolicy() >= 1) CutDataBlock(key, klen, true);
  }
  if (o_.filter_policy && klen >= 8) {                                  // block_based_table_builder.cc:514-528
    const int fl = docdb_filter_prefix_len(key, static_cast<int>(klen - 8));
    if (fl > 0 && (num_entries_ == 0 || last_filter_key_.size() != static_cast<size_t>(fl) || memcmp(last_filter_key_.data(), key, fl) != 0)) {
      if (filter_keys_ >= fg_.max_keys) FlushFilter(key, fl, true);
      filter_keys_++;
      uint32_t h = leveldb_hash(key, static_cast<uint32_t>(fl), kBloomSeed);   // AddHash, bloom.cc:43-61
      const uint32_t delta = (h >> 17) | (h << 15);
      const size_t b = static_cast<size_t>(h % fg_.num_lines) * kBloomLineBits;
      for (uint32_t i = 0; i < fg_.num_probes; i++) {
        const size_t bitpos = b + (h % kBloomLineBits);
        filter_bits_[bitpos / 8] = static_cast<char>(filter_bits_[bitpos / 8] | (1 << (bitpos % 8)));
        h += delta;
      }
      last_filter_key_.assign(reinterpret_cast<const char*>(key), fl);
    }
  }
  last_key_.assign(reinterpret_cast<const char*>(key), klen);
  block_.Add(key, klen, val, vlen);
  num_entries_++; raw_key_ += klen; raw_val_ += vlen;
  const uint8_t t = key[klen - 8];
  if (t == 0 || t == 7) deleted_keys_++;
}

void SplitSstWriter::CutDataBlock(const uint8_t* next_key, size_t next_len, bool has_next) {
  if (!block_.empty()) {
    AppendBlockTo(block_.Finish(), &data_, &pending_, o_.compression);
    block_.Reset();
    data_size_ += pending_.size + kTrailer;
  }
  num_data_blocks_++;
  metaw_.AddDataBlock(&last_key_, next_key, next_len, has_next, pending_);
}

void SplitSstWriter::FlushFilter(const uint8_t* next_key, size_t next_len, bool has_next) {
  const size_t bits_bytes = fg_.filter_bytes - 5;
  filter_bits_[bits_bytes] = static_cast<char>(fg_.num_probes);
  memcpy(&filter_bits_[bits_bytes + 1], &fg_.num_lines, 4);
  metaw_.AddFilterBlock(reinterpret_cast<const uint8_t*>(filter_bits_.data()), filter_bits_.size(), &last_filter_key_, next_key, next_len, has_next);
  filter_bits_.assign(fg_.filter_bytes, '\0');
  filter_keys_ = 0;
}

void SplitSstWriter::Finish() {
  if (!block_.empty()) CutDataBlock(nullptr, 0, false);
  if (o_.filter_policy) FlushFilter(nullptr, 0, false);
  MetaProps mp;
  mp.raw_key_size = raw_key_; mp.raw_value_size = raw_val_; mp.data_size = data_size_; mp.num_entries = num_entries_;
  mp.num_data_blocks = num_data_blocks_; mp.deleted_keys = deleted_keys_;
  metaw_.Finish(mp);
}


// ---------------------------------------------------------------------------------------------
// Concatenation of finished split SSTs with ascending, disjoint key ranges (the per-range outputs of a
// compaction run as subcompactions) into one table: see host_sst.h. Index keys inside a piece are
// reused; only the entry of a piece's LAST block (a short successor of its last key when the piece
// was written: index_builder.cc:72-77) is recomputed as the separator between the piece's largest key
// and the next piece's smallest, and likewise the index key of its last filter block.
static uint64_t PropVarint(const SstMeta& m, const char* name) {
  auto it = m.properties.find(name);
  if (it == m.properties.end()) return 0;
  const uint8_t* p = reinterpret_cast<const uint8_t*>(it->second.data());
  uint64_t v = 0;
  if (!ReadVarint(&p, p + it->second.size(), &v)) return 0;
  return v;
}

ConcatBuilder::ConcatBuilder(const TableOptions& o) : o_(o), w_(new MetaFileWriter(o)), mp_(new MetaProps()) {}
ConcatBuilder::~ConcatBuilder() { delete w_; delete mp_; }
void ConcatBuilder::Reserve(size_t bytes) { w_->Reserve(bytes); }

std::string ConcatBuilder::AddPiece(const SstPiece& piece, const SstPiece* next, const SstMeta* parsed) {
  try {
    SstMeta local;
    if (!parsed) {
      std::string e = ParseSplitSstMeta(piece.meta, piece.meta_len, &local);
      if (!e.empty()) return "piece " + std::to_string(n_pieces_) + ": " + e;
      parsed = &local;
    }
    const SstMeta& m = *parsed;
    const std::string tag = "piece " + std::to_string(n_pieces_);
    if (m.data_blocks.empty()) return tag + " has no data blocks";
    if (m.key_encoding != o_.key_encoding) return "pieces use a different data block key encoding than the output table options";
    if ((o_.filter_policy != 0) != !m.filter_blocks.empty()) return "filter blocks of " + tag + " do not match the output table options";
    if (o_.filter_policy && m.filter_policy_name != "DocKeyV3Filter") return "unknown filter policy " + m.filter_policy_name;
    if (piece.smallest.size() < 8 || piece.largest.size() < 8 || (next && next->smallest.size() < 8)) return "piece boundary keys are missing";
    if (n_pieces_ && CompareBytes(prev_largest_.substr(0, prev_largest_.size() - 8), piece.smallest.substr(0, piece.smallest.size() - 8)) >= 0)
      return "pieces are not in ascending, disjoint key order";
    if (next && CompareBytes(piece.largest.substr(0, piece.largest.size() - 8), next->smallest.substr(0, next->smallest.size() - 8)) >= 0)
      return "pieces are not in ascending, disjoint key order";
    const Handle& last = m.data_blocks.back();
    if (last.offset + last.size + kTrailer > piece.data_len) return tag + ": data file shorter than its index says";
    const bool last_piece = next == nullptr;
    // filter blocks of this piece first: the order of blocks inside the metadata file is free, the handles
    // in the filter index are what readers follow
    for (size_t f = 0; f < m.filter_blocks.size(); f++) {
      std::string key = m.filter_index_keys[f];
      if (f + 1 == m.filter_blocks.size() && !last_piece) {
        const std::string& lk = piece.largest; const std::string& nk = next->smallest;
        const int fl = docdb_filter_prefix_len(reinterpret_cast<const uint8_t*>(lk.data()), static_cast<int>(lk.size() - 8));
        const int fn = docdb_filter_prefix_len(reinterpret_cast<const uint8_t*>(nk.data()), static_cast<int>(nk.size() - 8));
        if (fl <= 0 || fn <= 0) return "a piece boundary key has no bloom filter key (not a DocKey): cannot place the filter index entry";
        key.assign(lk.data(), fl);
        ShortenUserSeparator(&key, reinterpret_cast<const uint8_t*>(nk.data()), static_cast<size_t>(fn));
      }
      w_->AddFilterBlockRaw(piece.meta + m.filter_blocks[f].offset, m.filter_blocks[f].size, key);
    }
    for (size_t b = 0; b < m.data_blocks.size(); b++) {
      const bool last_block = b + 1 == m.data_blocks.size();
      Handle h = m.data_blocks[b];
      h.offset += base_;
      if (last_block && !last_piece) {
        std::string key = piece.largest;
        InternalSeparator(&key, reinterpret_cast<const uint8_t*>(next->smallest.data()), next->smallest.size());
        w_->AddDataBlockRaw(key, true, h);
      } else {
        w_->AddDataBlockRaw(m.separators[b], !(last_block && last_piece), h);
      }
    }
    base_ += piece.data_len;
    mp_->raw_key_size += PropVarint(m, "rocksdb.raw.key.size");
    mp_->raw_value_size += PropVarint(m, "rocksdb.raw.value.size");
    mp_->num_entries += PropVarint(m, "rocksdb.num.entries");
    mp_->num_data_blocks += PropVarint(m, "rocksdb.num.data.blocks");
    mp_->deleted_keys += PropVarint(m, "rocksdb.deleted.keys");
    prev_largest_ = piece.largest;
    n_pieces_++;
    return std::string();
  } catch (const std::exception& ex) {
    return ex.what();
  }
}

std::string ConcatBuilder::Finish(std::string* meta_out) {
  try {
    if (!n_pieces_) return "no pieces";
    mp_->data_size = base_;
    w_->Finish(*mp_);
    w_->TakeMetaFile(meta_out);
    return std::string();
  } catch (const std::exception& ex) {
    return ex.what();
  }
}

std::string ConcatSplitSstMeta(const TableOptions& o, const std::vector<SstPiece>& pieces, std::string* meta_out) {
  try {
    std::vector<SstMeta> metas(pieces.size());
    {
      // the pieces' indexes are walked side by side (a 30 GB table has ~10^6 index entries)
      std::vector<std::string> errs(pieces.size());
      std::vector<std::thread> pool;
      for (size_t i = 0; i < pieces.size(); i++)
        pool.emplace_back([&, i] { errs[i] = ParseSplitSstMeta(pieces[i].meta, pieces[i].meta_len, &metas[i]); });
      for (std::thread& t : pool) t.join();
      for (size_t i = 0; i < pieces.size(); i++)
        if (!errs[i].empty()) return "piece " + std::to_string(i) + ": " + errs[i];
    }
    uint64_t total_meta = 0;
    for (size_t i = 0; i < pieces.size(); i++) total_meta += pieces[i].meta_len;
    ConcatBuilder cb(o);
    cb.Reserve(total_meta + total_meta / 4 + 65536);
    for (size_t i = 0; i < pieces.size(); i++) {
      std::string e = cb.AddPiece(pieces[i], i + 1 < pieces.size() ? &pieces[i + 1] : nullptr, &metas[i]);
      if (!e.empty()) return e;
    }
    return cb.Finish(meta_out);
  } catch (const std::exception& ex) {
    return ex.what();
  }
}

}  // namespace host
}  // namespace ybgpu
