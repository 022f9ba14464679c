// dev_logic.cuh — per-entry device logic of the H100 compaction engine.
//
// Everything here is __host__ __device__ so the same code that runs inside the sm_90a kernels
// (engine.cu) can be unit-tested on the CPU by tests/host_harness (this container has no GPU).
// The product never executes these functions on the host.
//
// Data model. Every input entry is decoded once (k_decode) into a fixed-stride "key record":
//
//   [0, S-16)   user key bytes, zero padded          (S = record stride, multiple of 16)
//   [S-16, S-8) u64  internal-key suffix (seq << 8 | type)   rocksdb/db/dbformat.cc:42-46
//   [S-8,  S-6) u16  user key length
//   [S-6]       u8   first byte of the value (0 if empty)     dockv/value_type.h:336-338
//   [S-5]       u8   flags (REC_F_*)
//   [S-4,  S)   u32  value length
//
// Zero padding + explicit length gives memcmp-with-length semantics (util/comparator.cc:37-47):
// compare padded words up to the longer length, then the shorter key is smaller.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define YB_HD __host__ __device__ __forceinline__
#define YB_HD_NOINLINE __host__ __device__ __noinline__ inline
#else
#define YB_HD inline
#define YB_HD_NOINLINE inline
#endif

namespace ybgpu {

enum : uint8_t {
  REC_F_HT_FILTERED = 0x80,   // invisible: file's HybridTime filter (docdb_rocksdb_util.cc:525-540)
  REC_F_OUT_OF_RANGE = 0x40,  // invisible: outside the job's key range (subcompaction / key-range shard). Table tombstones
                              // (`id ! # HT`) of the table the range starts in are loaded out of range on purpose: they
                              // seed slot 0 of the overwrite stack (docdb_compaction_context.cc:999-1024) and nothing else
  REC_F_INVISIBLE = 0xC0,
};

enum DevError : int {
  DEV_OK = 0,
  DEV_ERR_BAD_BLOCK = 1,          // block shorter than its restart array / bad restart offsets
  DEV_ERR_BAD_ENTRY = 2,          // entry header overruns its restart interval
  DEV_ERR_COMPRESSED = 3,         // trailer type byte != kNoCompression
  DEV_ERR_KEY_TOO_LONG = 4,
  DEV_ERR_IRREGULAR_RESTARTS = 5, // restart intervals of different sizes inside one file
  DEV_ERR_BAD_KEY = 6,            // DocKey / SubDocKey component decode failed
  DEV_ERR_UNSUPPORTED_KEY = 7,    // vector-index metadata keys, frozen containers nested deeper than 4
  DEV_ERR_TILE_OVERFLOW = 8,      // internal: a merge tile larger than its capacity (the host repartitions before this can happen)
  DEV_ERR_BAD_HT = 9,             // DocHybridTime at the end of a key is malformed
  DEV_ERR_BAD_VALUE = 10,         // value control fields malformed
  DEV_ERR_STACK_DEPTH = 11,       // more subkey levels than DEV_MAX_DEPTH
  DEV_ERR_UNSUPPORTED_VALUE = 12, // packed rows (need SchemaPackingProvider), merge/single-delete types
  DEV_ERR_BAD_CRC = 13,
  // 14 is retired: it was the per-tile limit on cotable / colocated tables, which no longer exists
  DEV_ERR_SHORT_KEY = 15,        // internal key shorter than 8 bytes
  DEV_ERR_UNSORTED = 16,          // input run not sorted
};

// ----------------------------------------------------------------------------------------------
// Little helpers
YB_HD uint32_t ld_u16(const uint8_t* p) { return static_cast<uint32_t>(p[0]) | (static_cast<uint32_t>(p[1]) << 8); }
YB_HD uint32_t ld_u32_unaligned(const uint8_t* p) {
  return static_cast<uint32_t>(p[0]) | (static_cast<uint32_t>(p[1]) << 8) | (static_cast<uint32_t>(p[2]) << 16) |
         (static_cast<uint32_t>(p[3]) << 24);
}
YB_HD uint64_t ld_u64_aligned(const uint8_t* p) { return *reinterpret_cast<const uint64_t*>(p); }
YB_HD uint64_t bswap64(uint64_t v) {
#if defined(__CUDA_ARCH__)
  uint32_t lo = static_cast<uint32_t>(v), hi = static_cast<uint32_t>(v >> 32);
  return (static_cast<uint64_t>(__byte_perm(lo, 0, 0x0123)) << 32) | __byte_perm(hi, 0, 0x0123);
#else
  return __builtin_bswap64(v);
#endif
}

// Record accessors (rec points at the start of an S-byte record).
YB_HD uint64_t rec_suffix(const uint8_t* rec, int S) { return ld_u64_aligned(rec + S - 16); }
YB_HD uint32_t rec_ulen(const uint8_t* rec, int S) { return *reinterpret_cast<const uint16_t*>(rec + S - 8); }
YB_HD uint8_t rec_vfirst(const uint8_t* rec, int S) { return rec[S - 6]; }
YB_HD uint8_t rec_flags(const uint8_t* rec, int S) { return rec[S - 5]; }
YB_HD uint32_t rec_vlen(const uint8_t* rec, int S) { return *reinterpret_cast<const uint32_t*>(rec + S - 4); }

// Compare user keys of two records: <0, 0, >0. Both zero padded, 8-byte aligned.
YB_HD int cmp_user_keys(const uint8_t* a, uint32_t la, const uint8_t* b, uint32_t lb) {
  uint32_t lmax = la > lb ? la : lb;
  uint32_t nw = (lmax + 7) >> 3;
  for (uint32_t w = 0; w < nw; w++) {
    uint64_t x = ld_u64_aligned(a + 8 * w), y = ld_u64_aligned(b + 8 * w);
    if (x != y) { return bswap64(x) < bswap64(y) ? -1 : 1; }
  }
  return la < lb ? -1 : (la > lb ? 1 : 0);
}

// Full internal-key order (rocksdb/db/dbformat.cc:92-114): user key ascending, suffix descending.
YB_HD int cmp_records(const uint8_t* a, const uint8_t* b, int S) {
  int r = cmp_user_keys(a, rec_ulen(a, S), b, rec_ulen(b, S));
  if (r) return r;
  uint64_t sa = rec_suffix(a, S), sb = rec_suffix(b, S);
  return sa > sb ? -1 : (sa < sb ? 1 : 0);
}

// Compare a key PREFIX (first g bytes of record p; bytes after g are ignored) with the user key
// of record c, as user keys. Used for DocKey-aligned partitioning.
YB_HD int cmp_prefix_vs_key(const uint8_t* p, uint32_t g, const uint8_t* c, uint32_t lc) {
  uint32_t lmax = g > lc ? g : lc;
  uint32_t nw = (lmax + 7) >> 3;
  for (uint32_t w = 0; w < nw; w++) {
    uint64_t x = 0;
    if (8 * w < g) {
      x = ld_u64_aligned(p + 8 * w);
      uint32_t valid = g - 8 * w;
      if (valid < 8) x &= (1ull << (8 * valid)) - 1;
    }
    uint64_t y = ld_u64_aligned(c + 8 * w);
    if (x != y) return bswap64(x) < bswap64(y) ? -1 : 1;
  }
  return g < lc ? -1 : (g > lc ? 1 : 0);
}

YB_HD uint32_t common_prefix_len(const uint8_t* a, uint32_t la, const uint8_t* b, uint32_t lb) {
  uint32_t m = la < lb ? la : lb;
  uint32_t i = 0;
  while (i + 8 <= m) {
    uint64_t x = ld_u64_aligned(a + i) ^ ld_u64_aligned(b + i);
    if (x) {
#if defined(__CUDA_ARCH__)
      return i + ((__ffsll(static_cast<long long>(x)) - 1) >> 3);
#else
      return i + (__builtin_ctzll(x) >> 3);
#endif
    }
    i += 8;
  }
  while (i < m && a[i] == b[i]) i++;
  return i;
}

// ----------------------------------------------------------------------------------------------
// util/fast_varint.cc:171-233 — signed "fast" varints (sign bit, unary length, magnitude).
YB_HD int fast_varint_size(const uint8_t* p, int n) {   // 0 on error
  if (n <= 0) return 0;
  uint32_t header = (static_cast<uint32_t>(p[0]) << 8) | (n > 1 ? p[1] : 0);
  if ((header & 0x8000) == 0) header ^= 0xffff;
  uint32_t x = (~header & 0x7fff) | 0x20;
#if defined(__CUDA_ARCH__)
  return __clz(static_cast<int>(x)) - 16;
#else
  return __builtin_clz(x) - 16;
#endif
}

YB_HD int fast_varint_decode(const uint8_t* p, int n, int64_t* out) {   // returns size, 0 on error
  int nb = fast_varint_size(p, n);
  if (nb == 0 || nb > n) return 0;
  const bool neg = (p[0] & 0x80) == 0;
  uint64_t negative = neg ? ~0ull : 0ull;
  uint64_t mask;
  switch (nb) {
    case 1: mask = 0x3full; break;           case 2: mask = 0x1fffull; break;
    case 3: mask = 0xfffffull; break;        case 4: mask = 0x7ffffffull; break;
    case 5: mask = 0x3ffffffffull; break;    case 6: mask = 0x1ffffffffffull; break;
    case 7: mask = 0xffffffffffffull; break; case 8: mask = 0x7fffffffffffffull; break;
    case 9: mask = 0x3fffffffffffffffull; break; default: mask = ~0ull; break;
  }
  uint64_t t = 0;
  for (int i = nb > 8 ? nb - 8 : 0; i < nb; i++) t = (t << 8) | p[i];
  *out = static_cast<int64_t>(((t & mask) | (~mask & negative)) - negative);
  return nb;
}

// Unsigned fast varint (fast_varint.cc:296-337).
YB_HD int fast_uvarint_decode(const uint8_t* p, int n, uint64_t* out) {
  if (n <= 0) return 0;
  uint32_t first = p[0];
  uint32_t x = (first << 1) ^ 0x1ff;
#if defined(__CUDA_ARCH__)
  int nb = __clz(static_cast<int>(x)) - 23 + 1;
#else
  int nb = __builtin_clz(x) - 23 + 1;
#endif
  if (n < nb) return 0;
  if (nb == 1) { *out = first & 0x7f; return 1; }
  uint64_t r = 0; int i = 0;
  if (nb == 9) {
    if (p[1] & 0x80) { nb = 10; r = p[1] & 0x3f; i = 2; }
    if (n < nb) return 0;
  } else { r = first & ((1u << (8 - nb)) - 1); i = 1; }
  for (; i < nb; i++) r = (r << 8) | p[i];
  *out = r;
  return nb;
}

YB_HD int fast_varint_encode(int64_t v, uint8_t* dest) {   // fast_varint.cc:73-150
  bool neg = v < 0;
  uint64_t uv = static_cast<uint64_t>(v);
  if (neg) uv = 1 + ~uv;
  int n = 1;
  for (uint64_t t = uv >> 6; t; t >>= 7) n++;
  int i;
  if (n == 10) { dest[0] = 0xff; dest[1] = 0xc0; i = 2; }
  else if (n == 9) { dest[0] = 0xff; dest[1] = static_cast<uint8_t>(0x80 | (uv >> 56)); i = 2; }
  else { dest[0] = static_cast<uint8_t>(~((1u << (8 - n)) - 1) | (uv >> (8 * (n - 1)))); i = 1; }
  for (; i < n; i++) dest[i] = static_cast<uint8_t>(uv >> (8 * (n - 1 - i)));
  if (neg) for (i = 0; i < n; i++) dest[i] = ~dest[i];
  return n;
}

YB_HD int fast_uvarint_encode(uint64_t v, uint8_t* dest) {   // fast_varint.cc:271-294
  int n = 1;
  for (uint64_t t = v >> 7; t; t >>= 7) n++;
  int i;
  if (n == 10) { dest[0] = 0xff; dest[1] = 0x80; i = 2; }
  else if (n == 9) { dest[0] = 0xff; dest[1] = static_cast<uint8_t>(v >> 56); i = 2; }
  else { dest[0] = static_cast<uint8_t>(~((1u << (9 - n)) - 1) | (v >> (8 * (n - 1)))); i = 1; }
  for (; i < n; i++) dest[i] = static_cast<uint8_t>(v >> (8 * (n - 1 - i)));
  return n;
}

// ----------------------------------------------------------------------------------------------
// common/doc_hybrid_time.cc. HT repr = (micros << 12) | logical (common/hybrid_time.h:68-97).
constexpr uint64_t kYbEpochMicros = 1500000000ull * 1000000;

// Length of the DocHybridTime at the end of a user key (doc_hybrid_time.cc:194-231); 0 on error.
YB_HD uint32_t doc_ht_len_from_end(const uint8_t* key, uint32_t ulen) {
  if (ulen == 0) return 0;
  uint32_t r = key[ulen - 1] & 0x1f;
  if (r < 1 || r > 30 || r >= ulen) return 0;
  return r;
}

// Decode an encoded DocHybridTime (doc_hybrid_time.cc:106-150) to the HybridTime repr.
YB_HD bool doc_ht_decode(const uint8_t* p, int n, uint64_t* ht) {
  int64_t v; int k;
  if (!(k = fast_varint_decode(p, n, &v))) return false;            // generation
  p += k; n -= k;
  if (!(k = fast_varint_decode(p, n, &v))) return false;
  int64_t micros = static_cast<int64_t>(kYbEpochMicros) + (-v);
  p += k; n -= k;
  if (!(k = fast_varint_decode(p, n, &v))) return false;
  int64_t logical = -v;
  p += k; n -= k;
  if (!(k = fast_varint_decode(p, n, &v))) return false;            // write id (ignored here)
  *ht = (static_cast<uint64_t>(micros) << 12) + static_cast<uint64_t>(logical);
  return true;
}

// Encode (doc_hybrid_time.cc:39-76).
YB_HD int doc_ht_encode(uint64_t ht, uint32_t write_id, uint8_t* dest) {
  uint8_t* out = dest;
  out += fast_varint_encode(0, out);
  out += fast_varint_encode(-static_cast<int64_t>((ht >> 12) - kYbEpochMicros), out);
  out += fast_varint_encode(-static_cast<int64_t>(ht & 0xfff), out);
  out += fast_varint_encode(-((static_cast<int64_t>(write_id) + 1) << 5), out);
  int size = static_cast<int>(out - dest);
  out[-1] = static_cast<uint8_t>((out[-1] & ~0x1f) | size);
  return size;
}

// Encoded DocHybridTime held by value (<= 30 bytes, doc_hybrid_time.h kMaxBytesPerEncodedHybridTime).
struct EncHt {
  uint8_t n;
  uint8_t b[31];
};
YB_HD void encht_set(EncHt* h, const uint8_t* p, uint32_t n) { h->n = static_cast<uint8_t>(n); for (uint32_t i = 0; i < n; i++) h->b[i] = p[i]; }
// Ordering of DocHybridTimes = REVERSED bytewise order of encodings (doc_hybrid_time.h:86-92):
// returns <0 if a is an EARLIER time than b.
YB_HD int encht_cmp(const uint8_t* a, uint32_t na, const uint8_t* b, uint32_t nb) {
  uint32_t m = na < nb ? na : nb;
  for (uint32_t i = 0; i < m; i++) {
    if (a[i] != b[i]) return a[i] < b[i] ? 1 : -1;     // reversed
  }
  return na < nb ? 1 : (na > nb ? -1 : 0);             // reversed length tie-break
}

// ----------------------------------------------------------------------------------------------
// Sizes of the comparable VarInt / Decimal encodings, which only the decoder can tell.
// util/varint.cc:159-205 (VarInt::DecodeFromComparable): after `reserved` reserved bits comes the
// sign bit, then a unary byte count, then the magnitude; negatives are stored complemented.
// `flip`: the caller's view of the bytes is complemented (a negative decimal's exponent).
YB_HD int comparable_varint_size(const uint8_t* p, int n, int reserved, bool flip) {
  if (n <= 0) return -DEV_ERR_BAD_KEY;
  const uint8_t fm = flip ? 0xff : 0x00;
  const bool negative = ((p[0] ^ fm) & (0x80u >> reserved)) == 0;
  const uint8_t m = negative ? static_cast<uint8_t>(~fm) : fm;
  const uint8_t first_or = reserved ? static_cast<uint8_t>(~((1u << (8 - reserved)) - 1u)) : 0;
  int idx = 0, ones = 0;
  uint8_t c = static_cast<uint8_t>((p[0] ^ m) | first_or);
  while (c == 0xff) {
    if (++idx >= n) return -DEV_ERR_BAD_KEY;              // "no prefix termination"
    ones += 8;
    c = static_cast<uint8_t>(p[idx] ^ m);
  }
  for (uint8_t t = 0x80; c & t; t >>= 1) ones++;
  ones -= reserved;
  if (ones > n) return -DEV_ERR_BAD_KEY;                  // "Not enough data in encoded varint"
  return ones;
}
// util/decimal.cc:339-367 (Decimal::DecodeFromComparable): 0x80 is zero; else the sign is the first
// bit (negatives complemented), the exponent a varint with two reserved bits, then mantissa digit
// pairs of which the last has its low bit clear.
YB_HD int comparable_decimal_size(const uint8_t* p, int n) {
  if (n <= 0) return -DEV_ERR_BAD_KEY;
  if (p[0] == 128) return 1;
  const bool flip = p[0] < 128;
  const int e = comparable_varint_size(p, n, 2, flip);
  if (e < 0) return e;
  for (int i = e; i < n; i++)
    if (!((flip ? ~p[i] : p[i]) & 1)) return i + 1;
  return -DEV_ERR_BAD_KEY;                                // "didn't find the ending"
}

// ----------------------------------------------------------------------------------------------
// dockv/primitive_value.cc:1232-1626 KeyEntryValue::DecodeKey(slice, nullptr): number of bytes of
// one key entry (type byte + payload) at p, or a negative DevError.
YB_HD_NOINLINE int key_entry_size_flat(const uint8_t* p, int n) {   // everything except frozen containers
  if (n <= 0) return -DEV_ERR_BAD_KEY;
  const uint8_t t = p[0];
  int fixed = -1;
  switch (t) {
    // value-less types (primitive_value.cc:750-765)
    case 6: case '%': case 'F': case 'i': case '~': case 0: case '|': case '$': case '&': case '\'':
    case 'T': case '{': case '3': case '4': case 'h':
      fixed = 0; break;
    case 'v': case 13: case 15: case 20: fixed = 1; break;                          // gin null, intent type sets
    case 'G': fixed = 2; break;                                                     // uint16 hash
    case 'H': case 'e': case '0': case 'g': case 'n': case 'O': case 'C': case 'M': fixed = 4; break;
    case 'I': case 'b': case '[': case 'U': case 'j': case 's': case 'c': case 'D': case 'L': fixed = 8; break;
    case 7: case 8: case 'V': fixed = 16; break;                                    // uuid-sized
    default: break;
  }
  if (fixed >= 0) return (n - 1 < fixed) ? -DEV_ERR_BAD_KEY : 1 + fixed;
  switch (t) {
    case 'S': case '\\': case '-': case 'x': case 'y': case '_': case 'o':          // zero-terminated strings (kBson: dockv/doc_bson.cc:33-35)
    case 'a': case ']': case '.': case '`': case 'p': {                             // complemented variants (kBsonDescending: :46-48)
      const uint8_t endb = (t == 'a' || t == ']' || t == '.' || t == '`' || t == 'p') ? 0xff : 0x00;
      int i = 1;
      if (i >= n) return -DEV_ERR_BAD_KEY;                  // "Encoded string is empty"
      for (;;) {
        // find the next terminator byte: bytewise to 8-byte alignment, then 8 bytes at a time
        while (i < n && p[i] != endb && (reinterpret_cast<uintptr_t>(p + i) & 7)) i++;
        if (i < n && p[i] != endb) {
          while (i + 8 <= n) {
            uint64_t w = ld_u64_aligned(p + i);
            if (endb) w = ~w;
            const uint64_t z = (w - 0x0101010101010101ull) & ~w & 0x8080808080808080ull;
            if (z) {
#if defined(__CUDA_ARCH__)
              i += (__ffsll(static_cast<long long>(z)) - 1) >> 3;
#else
              i += __builtin_ctzll(z) >> 3;
#endif
              break;
            }
            i += 8;
          }
          while (i < n && p[i] != endb) i++;
        }
        if (i >= n - 1) return -DEV_ERR_BAD_KEY;            // not terminated / single terminator byte
        if (p[i + 1] == endb) return i + 2;
        if (p[i + 1] != (endb ^ 1)) return -DEV_ERR_BAD_KEY;
        i += 2;
        if (i == n) return n;                               // doc_kv_util.cc:99 loop exit
      }
    }
    case 'K': case 'J': {                                   // column ids: fast signed varint
      int64_t v; int k = fast_varint_decode(p + 1, n - 1, &v);
      if (!k || v < 0 || v > 0x7fffffff) return -DEV_ERR_BAD_KEY;
      return 1 + k;
    }
    case '#': {                                             // hybrid time: 4 varints
      int i = 1;
      for (int j = 0; j < 4; j++) { int64_t v; int k = fast_varint_decode(p + i, n - i, &v); if (!k) return -DEV_ERR_BAD_KEY; i += k; }
      return i;
    }
    case '<': case '>':
      return -1000;                                         // frozen container: handled by key_entry_size
    case 'B': case 'f': {                                   // kVarInt / kVarIntDescending (primitive_value.cc:1334-1349)
      const int k = comparable_varint_size(p + 1, n - 1, 0, false);
      return k < 0 ? k : 1 + k;
    }
    case 'E': case 'd': {                                   // kDecimal / kDecimalDescending (:1314-1332)
      const int k = comparable_decimal_size(p + 1, n - 1);
      return k < 0 ? k : 1 + k;
    }
    default:
      return -DEV_ERR_BAD_KEY;
  }
}

// Full KeyEntryValue::DecodeKey size including frozen containers ('<' ... '!' / '>' ... '}'),
// which nest (primitive_value.cc:1287-1313). Iterative (no recursion: device stack is static).
YB_HD_NOINLINE int key_entry_size(const uint8_t* p, int n) {
  int k = key_entry_size_flat(p, n);
  if (k != -1000) return k;
  uint8_t endm[4];
  int depth = 0, i = 0;
  endm[depth++] = p[0] == '>' ? '}' : '!';
  i = 1;
  while (i < n) {
    if (p[i] == endm[depth - 1]) {
      i++;
      if (--depth == 0) return i;
      continue;
    }
    k = key_entry_size_flat(p + i, n - i);
    if (k == -1000) {
      if (depth >= 4) return -DEV_ERR_UNSUPPORTED_KEY;
      endm[depth++] = p[i] == '>' ? '}' : '!';
      i++;
      continue;
    }
    if (k < 0) return k;
    i += k;
  }
  return -DEV_ERR_BAD_KEY;   // "Reached end of slice looking for frozen group end marker"
}

YB_HD bool is_special_key_entry_type(uint8_t t) {   // value_type.h:280-284
  return t == 0 || t == '~' || t == 0xff || t == 13 || t == 21;
}

// One group of primitive values terminated by '!' (doc_key.cc:52-89). Returns bytes consumed.
YB_HD int consume_primitive_group(const uint8_t* p, int n) {
  int i = 0;
  for (;;) {
    if (i >= n) return -DEV_ERR_BAD_KEY;
    if (p[i] == '!') return i + 1;
    if (is_special_key_entry_type(p[i])) return -DEV_ERR_BAD_KEY;
    int k = key_entry_size(p + i, n - i);
    if (k < 0) return k;
    i += k;
  }
}

// Cotable / colocation id prefix size (doc_key.cc:1229-1270).
YB_HD int dockey_id_size(const uint8_t* p, int n) {
  if (n > 0 && p[0] == 'y') return n < 17 ? -DEV_ERR_BAD_KEY : 17;
  if (n > 0 && p[0] == '0') return n < 5 ? -DEV_ERR_BAD_KEY : 5;
  return 0;
}

// DocKey::EncodedSize(kWholeDocKey) of the bytes after the id prefix (doc_key.cc:543-590).
YB_HD int dockey_body_size(const uint8_t* p, int n, int* filter_end = nullptr) {
  // *filter_end (when asked for): end of the part DocDbAwareV3FilterPolicy keys the bloom filter by —
  // hashed components, or the first range component of a key without hash code
  // (DocKeyPart::kUpToHashOrFirstRange, doc_key.cc:523-538) — a by-product of this walk.
  int i = 0;
  bool hash_present = false;
  if (n > 0 && p[0] != '!') {
    if (is_special_key_entry_type(p[0])) return -DEV_ERR_BAD_KEY;
    if (p[0] == 'G') { if (n < 3) return -DEV_ERR_BAD_KEY; i = 3; hash_present = true; }
  }
  if (hash_present) { int k = consume_primitive_group(p + i, n - i); if (k < 0) return k; i += k; }
  if (filter_end) *filter_end = i;
  if (i >= n) return i;
  if (filter_end && !hash_present) {
    if (p[i] == '!') *filter_end = i + 1;
    else if (!is_special_key_entry_type(p[i])) { const int k1 = key_entry_size(p + i, n - i); *filter_end = k1 < 0 ? 0 : i + k1; }
  }
  int k = consume_primitive_group(p + i, n - i);
  if (k < 0) return k;
  return i + k;
}

// Length of the prefix that identifies the "row group" of a user key — the unit whose retention
// state is independent of every other group (docdb_compaction_context.cc:999-1003: state resets
// when fewer than 2 components are shared). Plain mode (no retention): the whole user key.
// Returns <0 DevError.
YB_HD int docdb_filter_prefix_len(const uint8_t* key, int ulen);
// filter_len (optional): the bloom filter key length of the same key (== docdb_filter_prefix_len), taken
// from the same DocKey walk where possible.
YB_HD int group_prefix_len(const uint8_t* key, int ulen, bool retention, int* filter_len = nullptr) {
  if (!retention) { if (filter_len) *filter_len = docdb_filter_prefix_len(key, ulen); return ulen; }
  if (ulen == 0) return -DEV_ERR_BAD_KEY;
  const uint8_t t = key[0];
  if (t == 10) { if (filter_len) *filter_len = docdb_filter_prefix_len(key, ulen); return ulen; }   // obsolete intent: dropped, any grouping is fine
  if (t == 6) return -DEV_ERR_UNSUPPORTED_KEY;       // vector index metadata: tablet-side filter
  int id = dockey_id_size(key, ulen);
  if (id < 0) return id;
  if (id > 0 && id < ulen && key[id] == '!') { if (filter_len) *filter_len = id + 1; return id + 1; }   // table tombstone: id ! # HT (doc_key.cc:973-982)
  int fe = 0;
  int body = dockey_body_size(key + id, ulen - id, filter_len ? &fe : nullptr);
  if (body < 0) return body;
  if (filter_len) *filter_len = id + fe;
  return id + body;
}

YB_HD int cmp_raw(const uint8_t* a, uint32_t la, const uint8_t* b, uint32_t lb) {
  const uint32_t m = la < lb ? la : lb;
  for (uint32_t i = 0; i < m; i++) if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
  return la < lb ? -1 : (la > lb ? 1 : 0);
}

// Key range of a range-sharded job: [lower, upper).
struct RangeDev { uint32_t lower_len, upper_len; uint8_t lower[256], upper[256]; };

// Retention parameters, precomputed on the host (docdb_compaction_context.cc:655-669).
struct RetentionDev {
  int enabled;
  uint64_t cutoff_ht;               // primary_cutoff_ht
  int64_t table_ttl_ns;
  EncHt cutoff_enc;                 // (cutoff, kMaxWriteId)
  int has_cotables_cutoff;          // HistoryCutoff::cotables_cutoff_ht set (master's sys catalog)
  uint64_t cotables_cutoff_ht;
  EncHt cotables_cutoff_enc;
  EncHt min_other_enc;              // (retain_delete_markers ? kMin : other_min, kMinWriteId)
  EncHt ht_min_enc;                 // DocHybridTime::kMin
  uint32_t lower_len, upper_len;    // key bounds
  uint8_t lower[256], upper[256];
};

constexpr int DEV_MAX_DEPTH = 24;
constexpr int64_t kMaxTtlNs = 0x7fffffffffffffffll;

struct Expiration { int64_t ttl_ns; uint64_t write_ht; };
struct Overwrite { EncHt ht; Expiration exp; };

// Decision for one entry.
enum : uint8_t {
  ENT_KEEP = 1,            // forwarded to the output
  ENT_ZERO_SEQ = 2,        // PrepareOutput zeroed the seqno (compaction_iterator.cc:476-482)
  ENT_VAL_TOMBSTONE = 4,   // value replaced by "X" (expired in a minor compaction, :1275-1277)
  ENT_VAL_REENCODE = 8,    // control fields re-encoded (TTL merge / intent doc-HT strip, :1278-1307)
  ENT_COUNTED = 16,        // counted as an input record (not HT-filtered)
  ENT_DROP_HIDDEN = 32,    // rule A
  ENT_DROP_OBSOLETE = 64,  // bottommost kTypeDeletion
  ENT_FIRST_OF_ROW = 128,  // first surviving entry of its DocKey (within a merge tile): the entry DocDBCompactionFeed passes
                           // to UpdateBoundaryValues (docdb_compaction_context.cc:754-773). Same bit as the merge kernel's
                           // tile-local group-start mark, which it replaces once the row groups are laid out.
};

// Re-encoded value prefix for ENT_VAL_REENCODE: new value = prefix[0..prefix_len) + old value
// from byte `skip` on (dockv/value.cc:118-132 AppendEncoded + rest of the value).
struct ValueRewrite { uint8_t prefix_len; uint8_t skip; uint8_t prefix[30]; };

// State of DocDBCompactionFeed restricted to one row group (prev_key_ is referenced, not copied:
// it always equals the first prev_len bytes of an earlier record of the same tile).
struct FeedState {
  const uint8_t* prev_key; uint32_t prev_len;
  uint32_t n_ends; uint32_t ends[DEV_MAX_DEPTH];
  uint32_t n_ow; Overwrite ow[DEV_MAX_DEPTH];
  bool within_merge_block;
};

YB_HD void feed_state_reset(FeedState* s) { s->prev_key = nullptr; s->prev_len = 0; s->n_ends = 0; s->n_ow = 0; s->within_merge_block = false; }
// State of the reference feed when it reaches a row of cotable / colocation id `id` after that
// table's tombstone entries (id ! # HT) were processed: prev_key_ = the id bytes, one component
// end, and slot 0 of the overwrite stack = the table-level overwrite (docdb_compaction_context.cc:
// 999-1024: slot 0 survives row changes, only new_stack_size == 1 entries replace it).
YB_HD void feed_state_seed(FeedState* s, const uint8_t* key, uint32_t id_len, const Overwrite& ow0) {
  s->prev_key = key; s->prev_len = id_len; s->n_ends = 1; s->ends[0] = id_len; s->n_ow = 1; s->ow[0] = ow0; s->within_merge_block = false;
}

// dockv/value.cc:77-115 DecodeControlFields over the head of a value. `v`/`n` is the value (the
// caller guarantees at least min(n, 64) readable bytes). Returns the control-field byte count or
// <0 on error.
struct ControlFields { uint64_t merge_flags; int64_t ttl_ns; int64_t timestamp; bool has_timestamp; uint32_t intent_ht_off, intent_ht_len; };
YB_HD int decode_control_fields(const uint8_t* v, int n, ControlFields* cf) {
  cf->merge_flags = 0; cf->ttl_ns = kMaxTtlNs; cf->has_timestamp = false; cf->timestamp = 0; cf->intent_ht_off = 0; cf->intent_ht_len = 0;
  int i = 0;
  if (n == 0) return 0;
  if (v[i] == 'k') {
    i++; int k = fast_uvarint_decode(v + i, n - i, &cf->merge_flags); if (!k) return -DEV_ERR_BAD_VALUE; i += k;
  }
  if (i < n && v[i] == '#') {
    i++; int start = i;
    for (int j = 0; j < 4; j++) { int k = fast_varint_size(v + i, n - i); if (k == 0 || i + k > n) return -DEV_ERR_BAD_VALUE; i += k; }
    cf->intent_ht_off = start; cf->intent_ht_len = i - start;
  }
  if (i < n && v[i] == 't') {
    i++; int64_t ms; int k = fast_varint_decode(v + i, n - i, &ms); if (!k) return -DEV_ERR_BAD_VALUE; i += k;
    cf->ttl_ns = ms * 1000000;
  }
  if (i < n && v[i] == 'u') {
    i++; if (n - i < 8) return -DEV_ERR_BAD_VALUE;
    uint64_t be = 0; for (int j = 0; j < 8; j++) be = (be << 8) | v[i + j];
    cf->timestamp = static_cast<int64_t>(be); cf->has_timestamp = true; i += 8;
  }
  return i;
}

// HybridTimeFilteringIterator::Satisfied (docdb/docdb_rocksdb_util.cc:525-565), negated: is this entry hidden by its
// input file's HybridTime filters? `global` = the file's global filter (HT_FILTER_NONE = none): hidden above it. Then the
// per-database cotable filters (master sys catalog after a restore: `n` sorted database oids with a hybrid time each,
// the tail of user_filter_data, :503-509): a key of a cotable ('y' + 16-byte comparable uuid, whose last four bytes are
// the database oid — the low half of the uuid is stored verbatim, util/uuid.cc:66-74,162-178) is hidden above the
// filter of its database; keys of other tables and databases without a filter stay visible. A key whose DocHybridTime
// does not decode is visible (:527-531).
constexpr uint64_t HT_FILTER_NONE = 0xfffffffffffffffeull;
YB_HD bool hidden_by_ht_filters(const uint8_t* key, uint32_t ulen, uint64_t global, const uint32_t* oids, const uint64_t* hts, uint32_t n) {
  const uint32_t htl = doc_ht_len_from_end(key, ulen);
  uint64_t ht;
  if (!htl || !doc_ht_decode(key + ulen - htl, htl, &ht)) return false;
  if (global != HT_FILTER_NONE && ht > global) return true;
  if (!n || ulen - htl < 17 || key[0] != 'y') return false;
  const uint32_t oid = static_cast<uint32_t>(key[13]) | (static_cast<uint32_t>(key[14]) << 8) | (static_cast<uint32_t>(key[15]) << 16) |
                       (static_cast<uint32_t>(key[16]) << 24);
  uint32_t lo = 0, hi = n;
  while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (oids[mid] < oid) lo = mid + 1; else hi = mid; }
  return lo < n && oids[lo] == oid && ht > hts[lo];
}

YB_HD bool has_control_fields(uint8_t first) { return first == 'k' || first == '#' || first == 't' || first == 'u'; }

// rocksdb/table/block.cc:65-87 DecodeEntry for kKeyDeltaEncodingSharedPrefix: parses the three
// varint32s at p (p < limit). Returns header length, 0 on error.
YB_HD int parse_entry_header(const uint8_t* p, uint32_t avail, uint32_t* shared, uint32_t* non_shared, uint32_t* vlen) {
  if (avail < 3) return 0;
  uint32_t a = p[0], b = p[1], c = p[2];
  if ((a | b | c) < 128) { *shared = a; *non_shared = b; *vlen = c; return 3; }
  if (avail >= 6) {
    // fields of at most two bytes (values below 16384: every key, most values): straight-line, no byte loop
    const uint32_t d = p[3], e = p[4], f = p[5];
    uint32_t i = 1, v0 = a, v1, v2;
    bool ok = true;
    if (a & 128) { ok = !(b & 128); v0 = (a & 127) | (b << 7); i = 2; }
    const uint32_t q0 = i == 1 ? b : c, q1 = i == 1 ? c : d;
    v1 = q0; uint32_t i1 = i + 1;
    if (q0 & 128) { ok = ok && !(q1 & 128); v1 = (q0 & 127) | (q1 << 7); i1 = i + 2; }
    const uint32_t r0 = i1 == 2 ? c : (i1 == 3 ? d : e), r1 = i1 == 2 ? d : (i1 == 3 ? e : f);
    v2 = r0; uint32_t i2 = i1 + 1;
    if (r0 & 128) { ok = ok && !(r1 & 128); v2 = (r0 & 127) | (r1 << 7); i2 = i1 + 2; }
    if (ok) { *shared = v0; *non_shared = v1; *vlen = v2; return static_cast<int>(i2); }
  }
  uint32_t out[3]; uint32_t i = 0;
  for (int f = 0; f < 3; f++) {
    uint32_t r = 0; int shift = 0; bool done = false;
    while (shift <= 28 && i < avail) {
      uint32_t byte = p[i++];
      if (byte & 128) r |= (byte & 127) << shift; else { r |= byte << shift; done = true; break; }
      shift += 7;
    }
    if (!done) return 0;
    out[f] = r;
  }
  *shared = out[0]; *non_shared = out[1]; *vlen = out[2];
  return static_cast<int>(i);
}

// rocksdb/table/block_internal.h:51-162 DecodeEntryThreeSharedParts for
// kKeyDeltaEncodingThreeSharedParts. Returns the header length (0 on error).
struct TspHeader {
  uint32_t shared_prefix, ns1, ns2, last_size, vlen;
  int64_t d1, d2;            // non_shared_{1,2}_size_delta
  uint64_t last_inc;         // 0 or 0x100 (seq + 1)
  bool something_shared;
};
YB_HD int tsp_get_varint(const uint8_t* p, uint32_t avail, uint64_t* out) {
  uint64_t r = 0; uint32_t i = 0;
  for (int shift = 0; shift <= 63 && i < avail; shift += 7) {
    const uint64_t b = p[i++];
    if (b & 128) r |= (b & 127) << shift; else { r |= b << shift; *out = r; return static_cast<int>(i); }
  }
  return 0;
}
YB_HD int parse_entry_header_tsp(const uint8_t* p, uint32_t avail, TspHeader* h) {
  if (avail < 2) return 0;
  uint64_t e1; int n = tsp_get_varint(p, avail, &e1);
  if (!n) return 0;
  uint32_t i = static_cast<uint32_t>(n);
  h->vlen = static_cast<uint32_t>(e1 >> 2);
  h->last_inc = (e1 & 2) << 7;
  h->shared_prefix = 0; h->ns1 = 0; h->ns2 = 0; h->last_size = 0; h->d1 = 0; h->d2 = 0;
  uint64_t v;
  if (e1 & 1) {
    n = tsp_get_varint(p + i, avail - i, &v); if (!n) return 0; i += n;
    h->shared_prefix = static_cast<uint32_t>(v); h->last_size = 8; h->something_shared = true; h->ns1 = 1; h->ns2 = 1;
    return static_cast<int>(i);
  }
  if (i >= avail) return 0;
  const uint8_t e2 = p[i++];
  if ((e2 & 1) == 0) {
    h->something_shared = false;
    if (e2 == 0) { n = tsp_get_varint(p + i, avail - i, &v); if (!n) return 0; i += n; h->ns1 = static_cast<uint32_t>(v); }
    else h->ns1 = e2 >> 1;
    return static_cast<int>(i);
  }
  h->something_shared = true;
  if ((e2 & 2) == 0) {
    h->last_size = 8; h->d2 = (e2 >> 2) & 1; h->ns1 = (e2 >> 3) & 7; h->ns2 = (e2 >> 6) & 3;
  } else {
    h->last_size = (e2 & 4) ? 8 : 0;
    n = tsp_get_varint(p + i, avail - i, &v); if (!n) return 0; i += n; h->ns1 = static_cast<uint32_t>(v);
    if (e2 & 8) { n = fast_varint_decode(p + i, static_cast<int>(avail - i), &h->d1); if (!n) return 0; i += n; }
    if (e2 & 16) { n = tsp_get_varint(p + i, avail - i, &v); if (!n) return 0; i += n; h->ns2 = static_cast<uint32_t>(v); }
    if (e2 & 32) { n = fast_varint_decode(p + i, static_cast<int>(avail - i), &h->d2); if (!n) return 0; i += n; }
  }
  n = tsp_get_varint(p + i, avail - i, &v); if (!n) return 0; i += n;
  h->shared_prefix = static_cast<uint32_t>(v);
  return static_cast<int>(i);
}
// Key length and the source offset of the shared middle (rocksdb/table/block.cc:313-343): returns
// false on corruption. prev_len = length of the previous key.
YB_HD bool tsp_key_layout(const TspHeader& h, uint32_t prev_len, uint32_t* klen, uint32_t* mid_src, uint32_t* mid_len) {
  if (!h.something_shared) { *klen = h.ns1; *mid_src = 0; *mid_len = 0; return true; }
  const int64_t prev_mid_start = static_cast<int64_t>(h.shared_prefix) + h.ns1 - h.d1;
  const int64_t prev_ns2 = static_cast<int64_t>(h.ns2) - h.d2;
  const int64_t except_mid = prev_mid_start + prev_ns2 + h.last_size;
  if (prev_mid_start < 0 || prev_ns2 < 0 || static_cast<int64_t>(prev_len) < except_mid) return false;
  const uint32_t mid = prev_len - static_cast<uint32_t>(except_mid);
  if (h.shared_prefix + mid + h.last_size == 0) return false;
  if (h.shared_prefix > prev_len) return false;
  *mid_src = static_cast<uint32_t>(prev_mid_start); *mid_len = mid;
  *klen = h.shared_prefix + h.ns1 + mid + h.ns2 + h.last_size;
  return true;
}

// ---- bloom filter (rocksdb/util/hash.cc:32-75, util/bloom.cc:43-61,384-455; docdb_filter_policy.cc) ----
// The LevelDB hash; tail bytes are added as signed chars (on-disk quirk the reference keeps).
YB_HD uint32_t leveldb_hash(const uint8_t* data, uint32_t n, uint32_t seed) {
  const uint32_t m = 0xc6a4a793u;
  uint32_t h = seed ^ (n * m);
  uint32_t i = 0;
  if ((reinterpret_cast<uintptr_t>(data) & 3) == 0) {          // records start 16-byte aligned: whole-word loads
    for (; i + 4 <= n; i += 4) { h += *reinterpret_cast<const uint32_t*>(data + i); h *= m; h ^= (h >> 16); }
  } else {
    for (; i + 4 <= n; i += 4) { h += ld_u32_unaligned(data + i); h *= m; h ^= (h >> 16); }
  }
  const uint32_t rest = n - i;
  if (rest == 3) h += static_cast<uint32_t>(static_cast<int32_t>(static_cast<int8_t>(data[i + 2])) << 16);
  if (rest >= 2) h += static_cast<uint32_t>(static_cast<int32_t>(static_cast<int8_t>(data[i + 1])) << 8);
  if (rest >= 1) { h += static_cast<uint32_t>(static_cast<int32_t>(static_cast<int8_t>(data[i]))); h *= m; h ^= (h >> 24); }
  return h;
}
constexpr uint32_t kBloomSeed = 0xbc9f1d34u;
constexpr uint32_t kBloomLineBits = 64 * 8;      // CACHE_LINE_SIZE * 8 (port/port_posix.h:179)

// Geometry of one fixed-size filter block (FixedSizeFilterBitsBuilder ctor, bloom.cc:389-422); the
// host computes it (double arithmetic as in the reference) and hands the integers to the device.
struct BloomGeometry { uint32_t num_lines, num_probes, max_keys, block_bytes, dev_stride; };   // dev_stride: 8-aligned pitch of a block on the device

// DocDbAwareV3FilterPolicy's key transformer: DocKey::EncodedSize(key, kUpToHashOrFirstRange)
// (doc_key.cc:417-422,523-590,1229-1310): cotable/colocation id, then either the hash code and the
// hashed components or, for range-partitioned keys, the first range component. 0 = not a DocKey
// (such keys are never added to the filter, docdb_filter_policy.cc:36-39).
YB_HD int docdb_filter_prefix_len(const uint8_t* key, int ulen) {
  const int id = dockey_id_size(key, ulen);
  if (id < 0) return 0;
  int i = id;
  bool hash_present = false;
  if (i < ulen && key[i] != '!') {
    if (is_special_key_entry_type(key[i])) return 0;
    if (key[i] == 'G') { if (ulen - i < 3) return 0; i += 3; hash_present = true; }
  }
  if (hash_present) { const int k = consume_primitive_group(key + i, ulen - i); if (k < 0) return 0; i += k; }
  if (i >= ulen || hash_present) return i;
  if (key[i] == '!') return i + 1;
  if (is_special_key_entry_type(key[i])) return 0;
  const int k = key_entry_size(key + i, ulen - i);
  return k < 0 ? 0 : i + k;
}

// ---- kKeyDeltaEncodingThreeSharedParts, encoder side -------------------------------------------
// (table/block_builder.cc:119-246,265-333; table/block_builder_internal.h:101-239.) Keys are given
// as (user key bytes, user key length, 8-byte suffix) so that a rewritten suffix (zeroed sequence
// number) never has to be materialised.
struct IKeyRef { const uint8_t* u; uint32_t ulen; uint64_t suffix; };
YB_HD uint8_t ikey_byte(const IKeyRef& k, uint32_t i) {
  return i < k.ulen ? k.u[i] : static_cast<uint8_t>(k.suffix >> (8 * (i - k.ulen)));
}
YB_HD int put_varint32_hd(uint8_t* p, uint32_t v) {
  int n = 0;
  while (v >= 128) { p[n++] = static_cast<uint8_t>(v | 128); v >>= 7; }
  p[n++] = static_cast<uint8_t>(v);
  return n;
}
YB_HD int put_varint64_hd(uint8_t* p, uint64_t v) {
  int n = 0;
  while (v >= 128) { p[n++] = static_cast<uint8_t>(v | 128); v >>= 7; }
  p[n++] = static_cast<uint8_t>(v);
  return n;
}
// FindMaxSharedSubstringAtTheSamePos (block_builder.cc:119-141): only runs ended by a mismatch count.
YB_HD void tsp_max_shared_same_pos(const IKeyRef& l, uint32_t lo, const IKeyRef& r, uint32_t ro, uint32_t n,
                                   uint32_t* best_off, uint32_t* best) {
  uint32_t b = 0, bo = 0, cur = 0;
  for (uint32_t i = 0; i < n; i++) {
    if (ikey_byte(l, lo + i) == ikey_byte(r, ro + i)) cur++;
    else { if (cur > b) { b = cur; bo = i - cur; } cur = 0; }
  }
  *best_off = bo; *best = b;
}
struct TspPlan {
  uint32_t shared;        // shared prefix
  uint32_t ns1, ns2;      // non-shared bytes stored: key[shared, shared+ns1) and key[klen-last_reuse-ns2, klen-last_reuse)
  uint32_t last_reuse;    // 0 or 8
  uint32_t hdr_len;
  uint8_t hdr[28];
};
// Plans the entry for `key` following `prev` (restart => no delta encoding; `shared` = common
// prefix of the two internal keys as plain byte strings, ignored on restarts).
YB_HD_NOINLINE void tsp_plan(const IKeyRef& prev, const IKeyRef& key, uint32_t vlen, bool restart, uint32_t shared, TspPlan* out) {
  const uint32_t pn = prev.ulen + 8, kn = key.ulen + 8;
  uint32_t prev_ns1 = pn, ns1 = kn, mid = 0, prev_ns2 = 0, ns2 = 0, last_reuse = 0;
  bool last_inc = false;
  if (restart) shared = 0;
  else {
    const uint32_t min_len = pn < kn ? pn : kn;
    if (min_len >= shared + 8) {                                     // CalculateLastInternalComponentReuse :222-246
      if (key.suffix == prev.suffix + 0x100) { last_inc = true; last_reuse = 8; }
      else if (key.suffix == prev.suffix) last_reuse = 8;
    }
    // FindMaxSharedMiddle :163-220 over prev[shared, pn - last_reuse) and key[shared, kn - last_reuse)
    const uint32_t ln = pn - shared - last_reuse, rn = kn - shared - last_reuse;
    uint32_t mo, ml; bool from_left = true; uint32_t min2;
    if (ln == rn) { min2 = rn; tsp_max_shared_same_pos(prev, shared, key, shared, min2, &mo, &ml); }
    else {
      uint32_t lso, rso;
      if (ln > rn) { min2 = rn; lso = shared + ln - min2; rso = shared; }
      else { min2 = ln; lso = shared; rso = shared + rn - min2; }
      tsp_max_shared_same_pos(prev, shared, key, shared, min2, &mo, &ml);
      uint32_t mo2, ml2;
      tsp_max_shared_same_pos(prev, lso, key, rso, min2, &mo2, &ml2);
      if (ml2 > ml) { from_left = false; mo = mo2; ml = ml2; }
    }
    if (ml == 0) { prev_ns1 = ln; ns1 = rn; }
    else if (from_left) { prev_ns1 = mo; ns1 = mo; mid = ml; prev_ns2 = ln - mo - ml; ns2 = rn - mo - ml; }
    else {
      const uint32_t mid_plus_ns2 = min2 - mo, t2 = mid_plus_ns2 - ml;
      prev_ns1 = ln - mid_plus_ns2; ns1 = rn - mid_plus_ns2; mid = ml; prev_ns2 = t2; ns2 = t2;
    }
  }
  (void)mid;
  // EncodeThreeSharedPartsSizes (block_builder_internal.h:101-239)
  const int64_t d1 = static_cast<int64_t>(ns1) - static_cast<int64_t>(prev_ns1);
  const int64_t d2 = static_cast<int64_t>(ns2) - static_cast<int64_t>(prev_ns2);
  const bool frequent = last_reuse > 0 && ns1 == 1 && ns2 == 1 && d1 == 0 && d2 == 0;
  uint8_t* h = out->hdr; int n = 0;
  n += put_varint64_hd(h + n, (static_cast<uint64_t>(vlen) << 2) | (static_cast<uint64_t>(last_inc) << 1) | (frequent ? 1u : 0u));
  if (frequent) n += put_varint32_hd(h + n, shared);
  else if (ns1 < kn) {                                               // something is reused
    if (last_reuse > 0 && d1 == 0 && (d2 == 0 || d2 == 1) && ns1 < 8 && ns2 < 4) {
      h[n++] = static_cast<uint8_t>(0b01 | ((d2 == 1) << 2) | (ns1 << 3) | (ns2 << 6));
    } else {
      h[n++] = static_cast<uint8_t>(0b11 | ((last_reuse > 0) << 2) | ((d1 != 0) << 3) | ((ns2 != 0) << 4) | ((d2 != 0) << 5));
      n += put_varint32_hd(h + n, ns1);
      if (d1 != 0) n += fast_varint_encode(d1, h + n);
      if (ns2 != 0) n += put_varint32_hd(h + n, ns2);
      if (d2 != 0) n += fast_varint_encode(d2, h + n);
    }
    n += put_varint32_hd(h + n, shared);
  } else {
    if (kn < 128 && kn > 0) h[n++] = static_cast<uint8_t>(kn << 1);
    else { h[n++] = 0; n += put_varint32_hd(h + n, kn); }
  }
  out->shared = shared; out->ns1 = ns1; out->ns2 = ns2; out->last_reuse = last_reuse; out->hdr_len = static_cast<uint32_t>(n);
}

YB_HD int encode_control_fields(const ControlFields& cf, uint8_t* out) {   // value.cc:118-132
  int i = 0;
  if (cf.merge_flags) { out[i++] = 'k'; i += fast_uvarint_encode(cf.merge_flags, out + i); }
  if (cf.ttl_ns != kMaxTtlNs) { out[i++] = 't'; i += fast_varint_encode(cf.ttl_ns / 1000000, out + i); }
  if (cf.has_timestamp) { out[i++] = 'u'; uint64_t v = static_cast<uint64_t>(cf.timestamp); for (int j = 7; j >= 0; j--) out[i++] = static_cast<uint8_t>(v >> (8 * j)); }
  return i;
}

// common/hybrid_time.cc:172-195.
YB_HD int compare_hts_to_delta(uint64_t begin, uint64_t end, int64_t delta_ns) {
  if (end < begin) return -1;
  uint64_t bn = (begin >> 12) * 1000, en = (end >> 12) * 1000, dn = static_cast<uint64_t>(delta_ns);
  if (en - bn > dn) return 1;
  if (en - bn == dn) { uint64_t bl = begin & 0xfff, el = end & 0xfff; return el > bl ? 1 : (el < bl ? -1 : 0); }
  return -1;
}

// One call of DocDBCompactionFeed::Feed (docdb_compaction_context.cc:941-1311) for the record
// `rec` (user key `ulen` bytes at rec). `val`/`vlen` give access to the value head (only read
// when the entry is at or below the history cutoff). Returns ENT_* bits (0 = dropped) or a
// negative DevError. `rw` is filled when ENT_VAL_REENCODE is returned.
YB_HD_NOINLINE int feed_step(FeedState* st, const RetentionDev& R, const uint8_t* key, uint32_t ulen,
                             uint8_t vfirst, const uint8_t* val, uint32_t vlen, ValueRewrite* rw) {
  if (ulen == 0) return -DEV_ERR_BAD_KEY;
  const uint8_t key_type = key[0];
  const bool is_sub_doc_key = !(key_type == 6 || key_type == 7);
  if (key_type == 10) return 0;                                                       // :951
  if (is_sub_doc_key && (R.lower_len || R.upper_len)) {                               // :955
    bool within = true;
    if (R.lower_len) {
      // key.compare(lower) >= 0, memcmp-with-length semantics on raw (unpadded) bounds
      uint32_t m = ulen < R.lower_len ? ulen : R.lower_len; int c = 0;
      for (uint32_t i = 0; i < m && !c; i++) c = static_cast<int>(key[i]) - static_cast<int>(R.lower[i]);
      if (!c) c = ulen < R.lower_len ? -1 : (ulen > R.lower_len ? 1 : 0);
      within = c >= 0;
    }
    if (within && R.upper_len) {
      uint32_t m = ulen < R.upper_len ? ulen : R.upper_len; int c = 0;
      for (uint32_t i = 0; i < m && !c; i++) c = static_cast<int>(key[i]) - static_cast<int>(R.upper[i]);
      if (!c) c = ulen < R.upper_len ? -1 : (ulen > R.upper_len ? 1 : 0);
      within = c < 0;
    }
    if (!within) return 0;
  }
  if (key_type == 6) return -DEV_ERR_UNSUPPORTED_KEY;

  // :972 same_bytes vs prev_key_
  uint32_t same = st->prev_len ? common_prefix_len(key, ulen, st->prev_key, st->prev_len) : 0;
  uint32_t shared;                                                                    // :977-989
  if (!same) shared = 0;
  else { shared = st->n_ends; while (shared > 0 && st->ends[shared - 1] > same) --shared; }
  st->n_ends = shared;                                                                // :1005
  if (is_sub_doc_key) {                                                               // :1008 (doc_key.cc:963-996)
    if (st->n_ends == 0) {
      int id = dockey_id_size(key, ulen);
      if (id < 0) return id;
      st->ends[st->n_ends++] = id;
    }
    uint32_t pos;
    if (st->n_ends == 1) {
      uint32_t id = st->ends[0];
      if (ulen < id + 1) return -DEV_ERR_BAD_KEY;
      if ((key[0] == '0' || key[0] == 'y') && key[id] == '!') {
        if (ulen < id + 2 || key[id + 1] != '#') return -DEV_ERR_BAD_KEY;
        pos = id + 1;
      } else {
        int body = dockey_body_size(key + id, ulen - id);
        if (body < 0) return body;
        pos = id + body;
        st->ends[st->n_ends++] = pos;
      }
    } else {
      pos = st->ends[st->n_ends - 1];
    }
    while (pos < ulen && key[pos] != '#') {                                          // DecodeSubkey doc_key.cc:827-838
      int k = key_entry_size(key + pos, ulen - pos);
      if (k < 0) return k;
      pos += k;
      if (st->n_ends >= DEV_MAX_DEPTH) return -DEV_ERR_STACK_DEPTH;
      st->ends[st->n_ends++] = pos;
    }
  } else {
    if (st->n_ends == 0) {                                                            // DecodeMetaSubKeyEnds :921-937
      int body = dockey_body_size(key, ulen);   // kTransactionApplyState handled as a DocKey
      if (body < 0) return body;
      st->ends[st->n_ends++] = body;
    }
  }
  const uint32_t new_stack = st->n_ends;
  if (shared < st->n_ow) st->n_ow = shared;                                           // :1021
  const uint32_t htl = doc_ht_len_from_end(key, ulen);                                // :1026
  if (!htl) return -DEV_ERR_BAD_HT;
  const uint8_t* ht = key + ulen - htl;
  EncHt prev_ow = st->n_ow ? st->ow[st->n_ow - 1].ht : R.ht_min_enc;                   // :1048
  const bool is_ttl_row = vlen > 0 && vfirst == 'k';                                  // :1066
  if (encht_cmp(ht, htl, prev_ow.b, prev_ow.n) < 0 && !is_ttl_row) return 0;          // :1067-1074
  Expiration last_exp; last_exp.ttl_ns = kMaxTtlNs; last_exp.write_ht = 0;
  if (st->n_ow) last_exp = st->ow[st->n_ow - 1].exp;
  while (st->n_ow + 1 < new_stack) {                                                  // :1078 (resize to new_stack-1)
    st->ow[st->n_ow].ht = prev_ow; st->ow[st->n_ow].exp = last_exp; st->n_ow++;
  }
  Expiration popped; popped.ttl_ns = kMaxTtlNs; popped.write_ht = 0;                  // :1083
  if (st->n_ow) popped = st->ow[st->n_ow - 1].exp;
  if (st->n_ow == new_stack) st->n_ow--;                                              // :1087
  if (same != st->ends[st->n_ends - 1]) st->within_merge_block = false;               // :1092
  // :1103-1114 — cotables on the master use their own cutoff
  const bool use_cot = key_type == 'y' && R.has_cotables_cutoff;
  const EncHt& chosen = use_cot ? R.cotables_cutoff_enc : R.cutoff_enc;
  const uint64_t chosen_ht = use_cot ? R.cotables_cutoff_ht : R.cutoff_ht;
  // LastExpiration() after the possible pop.
  Expiration cur_last; cur_last.ttl_ns = kMaxTtlNs; cur_last.write_ht = 0;
  if (st->n_ow) cur_last = st->ow[st->n_ow - 1].exp;

  if (encht_cmp(ht, htl, chosen.b, chosen.n) > 0) {                                   // :1117-1130
    st->prev_key = key; st->prev_len = st->ends[st->n_ends - 1];
    st->ow[st->n_ow].ht = prev_ow; st->ow[st->n_ow].exp = cur_last; st->n_ow++;
    if (vlen) {
      // ValueControlFields::Decode + packed-row check (:1123-1128). The value is only touched
      // when its first byte announces control fields; otherwise that byte IS the value type.
      uint8_t vtype = vfirst;
      if (has_control_fields(vfirst)) {
        ControlFields cf;
        uint32_t head = vlen < 64 ? vlen : 64;
        int c = decode_control_fields(val, head, &cf);
        if (c < 0) return c;
        vtype = static_cast<uint32_t>(c) < vlen ? val[c] : 0;
      }
      if (vtype == 'z' || vtype == '|') return -DEV_ERR_UNSUPPORTED_VALUE;
    }
    return ENT_KEEP;
  }

  ControlFields cf;
  int cfn = 0;
  if (vlen && has_control_fields(vfirst)) {
    uint32_t head = vlen < 64 ? vlen : 64;
    cfn = decode_control_fields(val, head, &cf);                                      // :1141
    if (cfn < 0) return cfn;
  } else {
    decode_control_fields(val, 0, &cf);   // defaults, does not touch val
  }
  // :1150-1210 need a SchemaPackingProvider (deleted columns / packing start): none => no-ops.
  const bool ow_is_prev = is_ttl_row || encht_cmp(prev_ow.b, prev_ow.n, ht, htl) > 0; // :1212
  const uint8_t value_type = cfn == 0 ? (vlen ? vfirst : 0) : (static_cast<uint32_t>(cfn) < vlen ? val[cfn] : 0);
  uint64_t this_ht = 0; bool this_ht_ok = false;
  Expiration expiration;                                                              // CalcExpiration :779-801
  if (st->within_merge_block) expiration = popped;
  else if (cf.ttl_ns == kMaxTtlNs && !is_ttl_row) expiration = cur_last;
  else {
    if (!doc_ht_decode(ht, htl, &this_ht)) return -DEV_ERR_BAD_HT;
    this_ht_ok = true;
    if (this_ht < cur_last.write_ht) expiration = cur_last;
    else { expiration.write_ht = this_ht; expiration.ttl_ns = cf.ttl_ns; }
  }
  if (ow_is_prev) st->ow[st->n_ow].ht = prev_ow; else encht_set(&st->ow[st->n_ow].ht, ht, htl);   // :1226
  st->ow[st->n_ow].exp = expiration; st->n_ow++;
  if (st->n_ow != new_stack) return -DEV_ERR_BAD_KEY;
  st->prev_key = key; st->prev_len = st->ends[st->n_ends - 1];                        // :1233
  const bool can_have_other_before = encht_cmp(ht, htl, R.min_other_enc.b, R.min_other_enc.n) >= 0;   // :775-777
  if (value_type == 'X' && !can_have_other_before) return 0;                          // :1246
  if (is_ttl_row) { st->within_merge_block = true; return 0; }                        // :1252
  int64_t true_ttl;                                                                   // ComputeTTL doc_ttl_util.cc:63-75
  if (expiration.ttl_ns != kMaxTtlNs) true_ttl = (expiration.ttl_ns / 1000000 == 0) ? kMaxTtlNs : expiration.ttl_ns;
  else true_ttl = R.table_ttl_ns;
  uint64_t key_ht;
  if (true_ttl == expiration.ttl_ns) key_ht = expiration.write_ht;
  else { if (!this_ht_ok) { if (!doc_ht_decode(ht, htl, &this_ht)) return -DEV_ERR_BAD_HT; this_ht_ok = true; } key_ht = this_ht; }
  bool has_expired = false;                                                           // doc_ttl_util.cc:25-31
  if (!(true_ttl == kMaxTtlNs || true_ttl == 0)) has_expired = compare_hts_to_delta(key_ht, chosen_ht, true_ttl) > 0;
  if (has_expired) {                                                                  // :1268-1277
    if (!can_have_other_before) return 0;
    return ENT_KEEP | ENT_VAL_TOMBSTONE;
  } else if (st->within_merge_block) {                                                // :1278-1293
    if (expiration.ttl_ns != kMaxTtlNs) {
      if (!this_ht_ok) { if (!doc_ht_decode(ht, htl, &this_ht)) return -DEV_ERR_BAD_HT; this_ht_ok = true; }
      int64_t diff_us = static_cast<int64_t>((st->ow[st->n_ow - 1].exp.write_ht >> 12) - (this_ht >> 12));
      expiration.ttl_ns += diff_us * 1000;
      st->ow[st->n_ow - 1].exp.ttl_ns = expiration.ttl_ns;
    }
    cf.ttl_ns = expiration.ttl_ns;
    rw->prefix_len = static_cast<uint8_t>(encode_control_fields(cf, rw->prefix));
    rw->skip = static_cast<uint8_t>(cfn);
    st->within_merge_block = false;
    return ENT_KEEP | ENT_VAL_REENCODE;
  } else if (value_type == 'z' || value_type == '|') {
    return -DEV_ERR_UNSUPPORTED_VALUE;                                                // packed rows :1294-1297
  } else if (cf.intent_ht_len) {                                                      // :1298-1307
    rw->prefix_len = static_cast<uint8_t>(encode_control_fields(cf, rw->prefix));
    rw->skip = static_cast<uint8_t>(cfn);
    return ENT_KEEP | ENT_VAL_REENCODE;
  }
  return ENT_KEEP;
}


// ----------------------------------------------------------------------------------------------
// Resuming DocDBCompactionFeed in the middle of a row group (merge tiles that start inside a group
// larger than a tile). Feed's state when it reaches a key K0 = (path components..., '#', HT) is a
// function of only those earlier entries whose component path is a PREFIX of K0's path — the
// ancestors `P_i # HT` (row-level / collection-level markers) and the earlier versions of K0's own
// SubDocKey: the overwrite stack is truncated to the shared components on every key change
// (docdb_compaction_context.cc:977-1021) and entries of sibling subtrees only write their own stack
// level or pad missing levels with the parent's value (:1078), which K0 would pad identically. All of
// these entries sort before K0 ('#' < every key entry type that can follow a component) and each
// level's entries are contiguous in every run, so a tile finds them with one search per run and
// level and replays them through feed_step — tiles stay independent, no state is carried between them.

// Component ends of a user key decoded from scratch: the same walk as feed_step's
// (SubDocKey::DecodeDocKeyAndSubKeyEnds, dockv/doc_key.cc:963-996). Returns the count or <0.
YB_HD int decode_key_ends(const uint8_t* key, uint32_t ulen, uint32_t* ends) {
  if (ulen == 0) return -DEV_ERR_BAD_KEY;
  const uint8_t key_type = key[0];
  int n = 0;
  if (key_type == 6 || key_type == 7) {
    const int body = dockey_body_size(key, ulen);
    if (body < 0) return body;
    ends[n++] = body;
    return n;
  }
  const int id = dockey_id_size(key, ulen);
  if (id < 0) return id;
  ends[n++] = id;
  if (ulen < static_cast<uint32_t>(id) + 1) return -DEV_ERR_BAD_KEY;
  uint32_t pos;
  if ((key[0] == '0' || key[0] == 'y') && key[id] == '!') {
    pos = id + 1;
  } else {
    const int body = dockey_body_size(key + id, ulen - id);
    if (body < 0) return body;
    pos = id + body;
    ends[n++] = pos;
  }
  while (pos < ulen && key[pos] != '#') {
    const int k = key_entry_size(key + pos, ulen - pos);
    if (k < 0) return k;
    pos += k;
    if (n >= DEV_MAX_DEPTH) return -DEV_ERR_STACK_DEPTH;
    ends[n++] = pos;
  }
  return n;
}

// (key[0, g) + extra) against the user key c: <0 / >0 as byte strings, 0 when c STARTS WITH the pattern.
// key and c are record pointers (zero padded, 8-byte aligned).
YB_HD int cmp_pattern(const uint8_t* key, uint32_t g, uint8_t extra, const uint8_t* c, uint32_t lc) {
  const uint32_t m = g < lc ? g : lc;
  const uint32_t cp = common_prefix_len(key, m, c, m);
  if (cp < m) return key[cp] < c[cp] ? -1 : 1;
  if (lc <= g) return 1;                               // c is a proper prefix of the pattern (or equals P): c < pattern
  return extra < c[g] ? -1 : (extra > c[g] ? 1 : 0);
}

struct ReplayRun { const uint8_t* rec; uint32_t limit; const uint8_t* data; const uint64_t* val_off; };
constexpr int REPLAY_MAX_RUNS = 64;

// First index in [0, run.limit] whose record is >= the pattern; the answer is usually close to the limit
// (inside the same group), so the search gallops backwards from there.
YB_HD uint32_t replay_lower_bound(const ReplayRun& run, int S, const uint8_t* key, uint32_t g) {
  uint32_t hi = run.limit, lo = 0, step = 1;
  while (hi > 0) {
    const uint32_t probe = hi > step ? hi - step : 0;
    const uint8_t* c = run.rec + static_cast<size_t>(probe) * S;
    if (cmp_pattern(key, g, '#', c, rec_ulen(c, S)) > 0) { lo = probe + 1; break; }   // rec[probe] < pattern
    hi = probe;
    if (probe == 0) break;
    step <<= 1;
  }
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    const uint8_t* c = run.rec + static_cast<size_t>(mid) * S;
    if (cmp_pattern(key, g, '#', c, rec_ulen(c, S)) > 0) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// One entry of a replay, in merged order: rule A against the entry replayed before it (*prev), deletions that are
// obsolete at the bottommost level skipped, every other entry fed. `val` = the value, needed only when its first byte
// announces control fields (nullptr otherwise). Returns 0 or a negative DevError.
YB_HD int replay_entry(FeedState* st, const RetentionDev& R, const uint8_t* rec, int S, const uint8_t* val,
                       const uint8_t** prev, int bottommost, uint64_t last_sequence) {
  const uint32_t cl = rec_ulen(rec, S);
  const bool hidden = *prev && cmp_user_keys(*prev, rec_ulen(*prev, S), rec, cl) == 0;   // rule A
  *prev = rec;
  if (hidden) return 0;
  const uint64_t suffix = rec_suffix(rec, S);
  if ((suffix & 0xff) == 0 && bottommost && (suffix >> 8) <= last_sequence) return 0;    // obsolete deletion
  ValueRewrite rw;
  const int d = feed_step(st, R, rec, cl, rec_vfirst(rec, S), val, rec_vlen(rec, S), &rw);
  return d < 0 ? d : 0;
}

// Replays, in merged order, the entries below runs[r].limit whose user key starts with key[0, g) + '#', except those
// whose flags intersect `skip`. The entries of one pattern are contiguous in every run: one galloping search per run,
// then a k-way merge of the k cursors. Returns 0 or a negative DevError.
YB_HD_NOINLINE int replay_pattern(FeedState* st, const RetentionDev& R, const ReplayRun* runs, int k, int S,
                                  const uint8_t* key, uint32_t g, uint8_t skip, int bottommost, uint64_t last_sequence) {
  uint32_t cur[REPLAY_MAX_RUNS];
  for (int r = 0; r < k; r++) cur[r] = replay_lower_bound(runs[r], S, key, g);
  const uint8_t* prev = nullptr;
  for (;;) {
    int best = -1; const uint8_t* bk = nullptr;
    for (int r = 0; r < k; r++) {
      if (cur[r] >= runs[r].limit) continue;
      const uint8_t* c = runs[r].rec + static_cast<size_t>(cur[r]) * S;
      if (cmp_pattern(key, g, '#', c, rec_ulen(c, S)) != 0) { cur[r] = runs[r].limit; continue; }   // left the pattern
      if (best < 0 || cmp_records(c, bk, S) < 0) { best = r; bk = c; }
    }
    if (best < 0) break;
    const uint32_t idx = cur[best]++;
    if (rec_flags(bk, S) & skip) continue;
    const uint8_t* val = nullptr;
    if (rec_vlen(bk, S) && has_control_fields(rec_vfirst(bk, S))) val = runs[best].data + runs[best].val_off[idx];
    const int d = replay_entry(st, R, bk, S, val, &prev, bottommost, last_sequence);
    if (d < 0) return d;
  }
  return 0;
}

// Brings *st (freshly reset, or seeded with the table tombstone state of a cotable) to the state Feed has
// when it reaches the record k0, which is the first record of a tile and lies inside a row group that
// began in an earlier tile. runs[r].limit = index of the first record of run r that belongs to this tile
// or a later one (everything below it sorts before k0). Returns 0 or a negative DevError.
YB_HD_NOINLINE int replay_ancestors(FeedState* st, const RetentionDev& R, const ReplayRun* runs, int k, int S,
                                    const uint8_t* k0, uint32_t ulen0, int bottommost, uint64_t last_sequence) {
  uint32_t ends[DEV_MAX_DEPTH];
  const int n = decode_key_ends(k0, ulen0, ends);
  if (n < 0) return n;
  const uint8_t t0 = k0[0];
  const bool sub_doc_key = !(t0 == 6 || t0 == 7);
  // level 0 of a SubDocKey is the table id: its entries are the table tombstones `id ! # HT`, which seed the rows
  // of the table elsewhere (table_seed / replay_table_seed). Only when k0 is itself such a tombstone are its earlier
  // versions replayed here: their pattern is id + '!' + '#'.
  const bool tombstone = sub_doc_key && n == 1;
  for (int lev = (sub_doc_key && !tombstone) ? 1 : 0; lev < n; lev++) {
    const uint32_t g = tombstone ? ends[0] + 1 : ends[lev];
    if (g >= ulen0) break;
    const int d = replay_pattern(st, R, runs, k, S, k0, g, REC_F_INVISIBLE, bottommost, last_sequence);
    if (d < 0) return d;
  }
  return 0;
}

// Cotable / colocated tables. The table tombstones `id ! # HT` sort before every row of their table and form one row
// group; Feed's slot 0 (the table-level overwrite) survives the row changes that follow (docdb_compaction_context.cc:
// 999-1024). After the tombstones of a table were replayed on a fresh *st (rule A, bottommost obsolete deletions
// skipped, HybridTime-filtered entries skipped, out-of-range ones INCLUDED: a key-range job that starts inside the
// table loads them for exactly this), table_seed turns *st into the state every row of the table starts from: slot 0
// kept (feed_state_seed) when the replay left a table-level overwrite, a reset state otherwise. `row` = a row key of
// the table, `id` = its id length.
YB_HD void table_seed(FeedState* st, const uint8_t* row, uint32_t id) {
  if (st->n_ow >= 1 && st->n_ends == 1) feed_state_seed(st, row, id, st->ow[0]);
  else feed_state_reset(st);
}

// The table tombstones of the table of `row` (id length `id`) replayed from the runs, below their limits, into *st,
// which then holds the state the table's rows start from (table_seed). Returns 0 or a negative DevError.
YB_HD_NOINLINE int replay_table_seed(FeedState* st, const RetentionDev& R, const ReplayRun* runs, int k, int S,
                                     const uint8_t* row, uint32_t id, int bottommost, uint64_t last_sequence) {
  alignas(8) uint8_t pattern[24] = {};                 // id + '!', zero padded (the id is 5 or 17 bytes)
  for (uint32_t q = 0; q < id; q++) pattern[q] = row[q];
  pattern[id] = '!';
  feed_state_reset(st);
  const int d = replay_pattern(st, R, runs, k, S, pattern, id + 1, REC_F_HT_FILTERED, bottommost, last_sequence);
  if (d < 0) return d;
  table_seed(st, row, id);
  return 0;
}

// ---- output check (V): what a reader finds in a finished data block ---------------------------------------------------
// The judgement of the device-side table check (verify_kernels.cuh), shared with the CPU tests: the walk of one restart
// interval the way BlockIter::ParseNextKey does it (table/block.cc:294-447), in either key encoding, with every key
// rebuilt, compared with its predecessor in InternalKeyComparator order (db/dbformat.cc:92-114) and handed to `expect`
// together with its value. Numbered like ybgpu_output_check::failure_kind.
enum VerifyKind : uint32_t {
  VERIFY_OK = 0, VERIFY_CHECKSUM = 1, VERIFY_COMPRESSED = 2, VERIFY_PARSE = 3, VERIFY_ORDER = 4, VERIFY_COUNT = 5,
  VERIFY_CONTENTS = 6, VERIFY_KEY_TOO_LONG = 7,
};
constexpr uint32_t VERIFY_MAX_IKEY = 1008 + 8;         // the engine's key limit: longer keys are not rebuilt

// First failure of a table: the lowest (block, entry) wins whatever the scheduling, so the three are packed into one word
// for atomicMin. ~0 = no failure.
YB_HD unsigned long long verify_pack(uint32_t block, uint32_t entry, uint32_t kind) {
  return (static_cast<unsigned long long>(block) << 32) | (static_cast<unsigned long long>(entry < 0x0fffffffu ? entry : 0x0fffffffu) << 4) | kind;
}

YB_HD int cmp_internal_keys(const uint8_t* a, uint32_t la, const uint8_t* b, uint32_t lb) {
  const int r = cmp_raw(a, la - 8, b, lb - 8);
  if (r) return r;
  uint64_t sa = 0, sb = 0;
  for (int i = 7; i >= 0; i--) { sa = (sa << 8) | a[la - 8 + i]; sb = (sb << 8) | b[lb - 8 + i]; }
  return sa > sb ? -1 : (sa < sb ? 1 : 0);
}

// The restart array of a block of `size` bytes (Block::Block / NumRestarts, table/block.cc:449-470): at least one restart
// point, the array inside the block. A data block without entries is never written (BlockBasedTableBuilder::Flush).
YB_HD bool verify_block_layout(const uint8_t* blk, uint32_t size, uint32_t* num_restarts, uint32_t* restarts_off) {
  if (size < 8) return false;
  const uint32_t nr = ld_u32_unaligned(blk + size - 4);
  if (nr == 0 || static_cast<uint64_t>(nr) * 4 + 4 > size) return false;
  *num_restarts = nr; *restarts_off = size - 4 - 4 * nr;
  return *restarts_off > 0;
}
// [*p, *end) of restart interval r: offsets ascend, the first is 0, the last interval ends at the restart array.
YB_HD bool verify_interval_bounds(const uint8_t* blk, uint32_t num_restarts, uint32_t restarts_off, uint32_t r, uint32_t* p, uint32_t* end) {
  *p = ld_u32_unaligned(blk + restarts_off + 4 * r);
  *end = r + 1 < num_restarts ? ld_u32_unaligned(blk + restarts_off + 4 * (r + 1)) : restarts_off;
  return (r != 0 || *p == 0) && *p < *end && *end <= restarts_off;
}

// The key of the entry at a restart point: it shares nothing, so its bytes are in the block itself. false = no such entry.
YB_HD bool verify_restart_key(const uint8_t* blk, uint32_t p, uint32_t end, int key_encoding, const uint8_t** key, uint32_t* klen) {
  uint32_t h, kl, vl;
  if (key_encoding == 2) {
    TspHeader th;
    h = static_cast<uint32_t>(parse_entry_header_tsp(blk + p, end - p, &th));
    if (!h || th.something_shared) return false;
    kl = th.ns1; vl = th.vlen;
  } else {
    uint32_t shared;
    h = static_cast<uint32_t>(parse_entry_header(blk + p, end - p, &shared, &kl, &vl));
    if (!h || shared) return false;
  }
  if (kl < 8 || static_cast<uint64_t>(p) + h + kl + vl > end) return false;
  *key = blk + p + h; *klen = kl;
  return true;
}

struct VerifyWalk {
  uint32_t n;                  // entries parsed before the walk ended
  uint32_t kind;               // VERIFY_OK or what stopped it, at entry n of the interval
  const uint8_t* last_key;     // the last key parsed (inside one of the two key buffers) and its length
  uint32_t last_klen;
};
struct VerifyNoExpect {        // a table with nothing to compare it with (ybgpu_sst_verify_device)
  YB_HD bool operator()(uint32_t, const uint8_t*, uint32_t, const uint8_t*, uint32_t) const { return true; }
};

// Entries [p, end) of one restart interval. buf0 / buf1: two key buffers of `kcap` bytes; expect(ordinal, key, klen,
// value, vlen) says whether entry `ordinal` = ord_base + position of the table is the one that belongs there. No byte
// outside [blk + p, blk + end) is read, whatever the block holds.
template <class Expect>
YB_HD void verify_interval(const uint8_t* blk, uint32_t p, uint32_t end, int key_encoding, uint8_t* buf0, uint8_t* buf1,
                                    uint32_t kcap, uint32_t ord_base, const Expect& expect, VerifyWalk* w) {
  uint8_t* cur = buf0; uint8_t* prev = buf1;
  uint32_t prev_klen = 0, n = 0, kind = VERIFY_OK;
  while (p < end) {
    uint32_t klen, vlen;
    if (key_encoding == 2) {
      TspHeader th; uint32_t ms, ml;
      const int h = parse_entry_header_tsp(blk + p, end - p, &th);
      if (!h || (n == 0 && th.something_shared) || !tsp_key_layout(th, prev_klen, &klen, &ms, &ml) ||
          static_cast<uint64_t>(p) + h + th.ns1 + th.ns2 + th.vlen > end || klen < 8) { kind = VERIFY_PARSE; break; }
      if (klen > kcap) { kind = VERIFY_KEY_TOO_LONG; break; }
      p += h;
      uint32_t o = 0;
      if (!th.something_shared) {
        for (; o < th.ns1; o++) cur[o] = blk[p + o];
      } else {
        uint64_t last = 0;
        if (th.last_size) { for (int i = 7; i >= 0; i--) last = (last << 8) | prev[prev_klen - 8 + i]; last += th.last_inc; }
        for (; o < th.shared_prefix; o++) cur[o] = prev[o];
        for (uint32_t i = 0; i < th.ns1; i++) cur[o++] = blk[p + i];
        for (uint32_t i = 0; i < ml; i++) cur[o++] = prev[ms + i];
        for (uint32_t i = 0; i < th.ns2; i++) cur[o++] = blk[p + th.ns1 + i];
        if (th.last_size) for (int i = 0; i < 8; i++) cur[o++] = static_cast<uint8_t>(last >> (8 * i));
      }
      p += th.ns1 + th.ns2;
      vlen = th.vlen;
    } else {
      uint32_t shared, non_shared;
      const int h = parse_entry_header(blk + p, end - p, &shared, &non_shared, &vlen);
      if (!h || shared > prev_klen || (n == 0 && shared != 0) || static_cast<uint64_t>(p) + h + non_shared + vlen > end ||
          shared + non_shared < 8) { kind = VERIFY_PARSE; break; }
      klen = shared + non_shared;
      if (klen > kcap) { kind = VERIFY_KEY_TOO_LONG; break; }
      p += h;
      for (uint32_t i = 0; i < shared; i++) cur[i] = prev[i];
      for (uint32_t i = 0; i < non_shared; i++) cur[shared + i] = blk[p + i];
      p += non_shared;
    }
    if (n > 0 && cmp_internal_keys(prev, prev_klen, cur, klen) >= 0) { kind = VERIFY_ORDER; break; }
    if (!expect(ord_base + n, cur, klen, blk + p, vlen)) { kind = VERIFY_CONTENTS; break; }
    p += vlen;
    uint8_t* t = cur; cur = prev; prev = t;
    prev_klen = klen;
    n++;
  }
  w->n = n; w->kind = kind; w->last_key = prev; w->last_klen = prev_klen;
}

}  // namespace ybgpu
