// TEST-ONLY: the device logic of yugabyte-db_b200/csrc/dev_logic.cuh run on the CPU, in merged order, with the rows of
// cotable / colocated tables seeded the way a merge tile seeds the table it starts in: slot 0 of the overwrite stack
// comes from replay_table_seed over the INPUT RUNS, each run cut where the row starts. Every row group of such a table
// takes that path here, so the lookup is exercised for every row against the oracle. Built and loaded by
// tests/test_colocated_cpu.py; not part of the product.
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "../../yugabyte-db_b200/csrc/dev_logic.cuh"

using namespace ybgpu;

namespace {
struct Out { std::string keys, vals; std::vector<uint64_t> koff{0}, voff{0}; };
Out* g_out = nullptr;
}

extern "C" {

// returns 0 or a positive DevError; same arguments as tests/host_harness/harness.cc hh_compact
int cs_compact(int n_runs, const uint64_t* run_start, const uint8_t* keys, const uint64_t* koff, const uint8_t* vals,
               const uint64_t* voff, int retention, uint64_t cutoff_ht, int64_t table_ttl_ns, int retain_markers,
               uint64_t other_min_ht, int bottommost, uint64_t last_sequence, const uint8_t* largest, uint64_t largest_len,
               const uint8_t* lower, uint64_t lower_len, const uint8_t* upper, uint64_t upper_len, uint64_t cotables_cutoff_ht) {
  delete g_out; g_out = new Out;
  const uint64_t n = run_start[n_runs];
  size_t max_ulen = 0;
  for (uint64_t i = 0; i < n; i++) max_ulen = std::max<size_t>(max_ulen, koff[i + 1] - koff[i] - 8);
  const int S = std::max<int>(32, static_cast<int>(((max_ulen + 16) + 15) & ~15ull));
  std::vector<uint8_t> store(static_cast<size_t>(n) * S + 64, 0);
  uint8_t* base = store.data();
  base += (16 - (reinterpret_cast<uintptr_t>(base) & 15)) & 15;
  for (uint64_t i = 0; i < n; i++) {
    uint8_t* r = base + i * S;
    const uint32_t ulen = static_cast<uint32_t>(koff[i + 1] - koff[i]) - 8, vlen = static_cast<uint32_t>(voff[i + 1] - voff[i]);
    memcpy(r, keys + koff[i], ulen);
    memcpy(r + S - 16, keys + koff[i] + ulen, 8);
    const uint16_t ul16 = static_cast<uint16_t>(ulen); memcpy(r + S - 8, &ul16, 2);
    r[S - 6] = vlen ? vals[voff[i]] : 0; r[S - 5] = 0;
    memcpy(r + S - 4, &vlen, 4);
  }
  std::vector<uint32_t> order(n);
  for (uint64_t i = 0; i < n; i++) order[i] = static_cast<uint32_t>(i);
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return cmp_records(base + size_t(a) * S, base + size_t(b) * S, S) < 0; });

  RetentionDev R{};
  R.enabled = retention; R.cutoff_ht = cutoff_ht; R.table_ttl_ns = table_ttl_ns;
  R.cutoff_enc.n = static_cast<uint8_t>(doc_ht_encode(cutoff_ht, 0xffffffffu, R.cutoff_enc.b));
  R.min_other_enc.n = static_cast<uint8_t>(doc_ht_encode(retain_markers ? 0 : other_min_ht, 0, R.min_other_enc.b));
  R.ht_min_enc.n = static_cast<uint8_t>(doc_ht_encode(0, 0, R.ht_min_enc.b));
  R.has_cotables_cutoff = cotables_cutoff_ht != 0xfffffffffffffffeull; R.cotables_cutoff_ht = cotables_cutoff_ht;
  if (R.has_cotables_cutoff) R.cotables_cutoff_enc.n = static_cast<uint8_t>(doc_ht_encode(cotables_cutoff_ht, 0xffffffffu, R.cotables_cutoff_enc.b));
  R.lower_len = static_cast<uint32_t>(lower_len); memcpy(R.lower, lower, lower_len);
  R.upper_len = static_cast<uint32_t>(upper_len); memcpy(R.upper, upper, upper_len);

  // slot 0 for a row of a cotable / colocated table: its tombstones replayed from the runs below the row
  auto seed_from_runs = [&](FeedState* st, const uint8_t* e, uint32_t id) -> int {
    std::vector<ReplayRun> rr(n_runs);
    for (int r = 0; r < n_runs; r++) {
      const uint8_t* rec = base + size_t(run_start[r]) * S;
      uint32_t lo = 0, hi = static_cast<uint32_t>(run_start[r + 1] - run_start[r]);
      while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (cmp_records(rec + size_t(mid) * S, e, S) < 0) lo = mid + 1; else hi = mid;
      }
      rr[r] = ReplayRun{rec, lo, vals, voff + run_start[r]};
    }
    const int d = replay_table_seed(st, R, rr.data(), n_runs, S, e, id, bottommost, last_sequence);
    return d < 0 ? -d : 0;
  };

  FeedState st; feed_state_reset(&st);
  const uint8_t* prev_group = nullptr; int prev_g = -1;
  const uint8_t* prev_rec = nullptr;
  for (uint64_t i = 0; i < n; i++) {
    const uint32_t id = order[i];
    const uint8_t* e = base + size_t(id) * S;
    const uint32_t ulen = rec_ulen(e, S);
    const int g = group_prefix_len(e, ulen, retention != 0);
    if (g < 0) return -g;
    if (!prev_group || g != prev_g || common_prefix_len(e, g, prev_group, g) < static_cast<uint32_t>(g)) {
      feed_state_reset(&st); prev_group = e; prev_g = g;
      if (retention && (e[0] == 'y' || e[0] == '0')) {
        const int tid = dockey_id_size(e, ulen);
        if (tid > 0 && static_cast<uint32_t>(tid) < ulen && e[tid] != '!') {
          const int rc = seed_from_runs(&st, e, static_cast<uint32_t>(tid));
          if (rc) return rc;
        }
      }
    }
    const bool first_occ = !prev_rec || cmp_user_keys(prev_rec, rec_ulen(prev_rec, S), e, ulen) != 0;   // rule A
    prev_rec = e;
    if (!first_occ) continue;
    uint64_t suffix = rec_suffix(e, S);
    if ((suffix & 0xff) == 0 && bottommost && (suffix >> 8) <= last_sequence) continue;
    if (bottommost && (suffix >> 8) < last_sequence && !(ulen == largest_len && memcmp(e, largest, ulen) == 0)) suffix &= 0xff;
    const uint8_t* val = vals + voff[id];
    const uint32_t vlen = rec_vlen(e, S);
    int d = ENT_KEEP;
    ValueRewrite rw{};
    if (retention) {
      d = feed_step(&st, R, e, ulen, rec_vfirst(e, S), has_control_fields(rec_vfirst(e, S)) ? val : nullptr, vlen, &rw);
      if (d < 0) return -d;
      if (d == 0) continue;
    }
    g_out->keys.append(reinterpret_cast<const char*>(e), ulen);
    g_out->keys.append(reinterpret_cast<const char*>(&suffix), 8);
    if (d & ENT_VAL_TOMBSTONE) g_out->vals.push_back('X');
    else if (d & ENT_VAL_REENCODE) {
      g_out->vals.append(reinterpret_cast<const char*>(rw.prefix), rw.prefix_len);
      g_out->vals.append(reinterpret_cast<const char*>(val + rw.skip), vlen - rw.skip);
    } else g_out->vals.append(reinterpret_cast<const char*>(val), vlen);
    g_out->koff.push_back(g_out->keys.size()); g_out->voff.push_back(g_out->vals.size());
  }
  return 0;
}

uint64_t cs_num() { return g_out->koff.size() - 1; }
const uint8_t* cs_keys() { return reinterpret_cast<const uint8_t*>(g_out->keys.data()); }
const uint8_t* cs_vals() { return reinterpret_cast<const uint8_t*>(g_out->vals.data()); }
const uint64_t* cs_koff() { return g_out->koff.data(); }
const uint64_t* cs_voff() { return g_out->voff.data(); }

}  // extern "C"
