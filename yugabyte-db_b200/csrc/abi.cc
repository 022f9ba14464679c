// abi.cc — extern "C" surface declared in include/ybgpu_compaction.h.
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "engine.h"
#include "host_sst.h"

using ybgpu::Engine;

struct ybgpu_job {
  std::unique_ptr<Engine> engine;
  // host copies of the results (filled lazily)
  bool have_kv = false;
  std::vector<uint8_t> keys, vals;
  std::vector<uint64_t> koff, voff;
  bool have_sst = false;
  // small per-block results of the GPU the host builds the metadata file from (fetched before the
  // big data-file copy is queued, so that they do not wait behind it on the copy engine)
  struct SstParts {
    bool fetched = false;
    uint64_t data_len = 0; uint32_t nb = 0, stride = 0;
    std::vector<uint64_t> off; std::vector<uint8_t> bnd;
    uint32_t nfb = 0, fbytes = 0, fstride = 0;
    std::vector<uint8_t> filters, fkeys; std::vector<uint32_t> ffirst, bfirst;
  } parts;
  std::string meta_file;
  uint64_t data_len = 0;
  uint64_t num_blocks = 0;
  std::string error;
};

static thread_local std::string g_last_error;

void ybgpu::JoinMemGroup(ybgpu_job* job, MemGroup* group) { job->engine->JoinMemGroup(group); }

static ybgpu_status JobFail(ybgpu_job* j, ybgpu_status s, const std::string& msg) {
  j->error = msg;
  return s;
}
static ybgpu_status Sync(ybgpu_job* j, ybgpu_status s) {
  if (s != YBGPU_OK) j->error = j->engine->error();
  return s;
}

extern "C" {

void ybgpu_job_options_init(ybgpu_job_options* o) {
  memset(o, 0, sizeof(*o));
  o->bottommost_level = 1;
  o->last_sequence = YBGPU_MAX_SEQUENCE;
  o->retention_enabled = 1;
  o->history_cutoff_ht = YBGPU_HT_MIN;
  o->cotables_cutoff_ht = YBGPU_HT_INVALID;
  o->table_ttl_ns = YBGPU_TTL_MAX_NS;
  o->other_min_ht = YBGPU_HT_MAX;
  o->block_size = 32 * 1024;
  o->block_restart_interval = 16;
  o->block_size_deviation = 10;
  o->output_key_encoding = YBGPU_KEY_ENCODING_SHARED_PREFIX;
  o->index_block_size = 32 * 1024;
  o->min_keys_per_index_block = 100;
  o->verify_checksums = 1;
  o->filter_policy = YBGPU_FILTER_NONE;
  o->filter_block_size = 64 * 1024;
}

ybgpu_status ybgpu_job_create(const ybgpu_job_options* options, ybgpu_job** job) {
  if (!options || !job) { g_last_error = "null argument"; return YBGPU_INVALID_ARGUMENT; }
  if (!ybgpu::host::OutputCompressionSupported(options->output_compression)) {
    g_last_error = ybgpu::host::UnsupportedOutputCompression(options->output_compression); return YBGPU_NOT_SUPPORTED;
  }
  std::unique_ptr<ybgpu_job> j(new ybgpu_job);
  j->engine.reset(new Engine(*options));
  ybgpu_status s = j->engine->Init();
  if (s != YBGPU_OK) { g_last_error = j->engine->error(); return s; }
  *job = j.release();
  return YBGPU_OK;
}

void ybgpu_job_destroy(ybgpu_job* job) { delete job; }
const char* ybgpu_job_error(const ybgpu_job* job) { return job ? job->error.c_str() : "null job"; }
const char* ybgpu_last_error(void) { return g_last_error.c_str(); }

ybgpu_status ybgpu_job_add_input(ybgpu_job* job, const uint8_t* data_file, uint64_t data_file_len,
                                 const ybgpu_block_handle* handles, uint64_t num_handles, int32_t key_encoding,
                                 uint64_t hybrid_time_filter) {
  if (!job) return YBGPU_INVALID_ARGUMENT;
  return Sync(job, job->engine->AddInput(data_file, data_file_len, handles, num_handles, key_encoding, hybrid_time_filter, false));
}

ybgpu_status ybgpu_job_add_input_kv(ybgpu_job* job, const uint8_t* keys, const uint64_t* key_offsets,
                                    const uint8_t* values, const uint64_t* value_offsets, uint64_t n) {
  if (!job) return YBGPU_INVALID_ARGUMENT;
  return Sync(job, job->engine->AddInputKv(keys, key_offsets, values, value_offsets, n));
}

ybgpu_status ybgpu_job_set_cotable_filters(ybgpu_job* job, const uint32_t* db_oids, const uint64_t* hybrid_times, uint32_t n) {
  if (!job) return YBGPU_INVALID_ARGUMENT;
  return Sync(job, job->engine->SetCotableFilters(db_oids, hybrid_times, n));
}

ybgpu_status ybgpu_job_wait_inputs(ybgpu_job* job) {
  if (!job) return YBGPU_INVALID_ARGUMENT;
  return Sync(job, job->engine->WaitInputs());
}

ybgpu_status ybgpu_job_add_input_device(ybgpu_job* job, const uint8_t* data_file_dev, uint64_t data_file_len,
                                        const ybgpu_block_handle* handles, uint64_t num_handles, int32_t key_encoding,
                                        uint64_t hybrid_time_filter) {
  if (!job) return YBGPU_INVALID_ARGUMENT;
  return Sync(job, job->engine->AddInput(data_file_dev, data_file_len, handles, num_handles, key_encoding, hybrid_time_filter, true));
}

ybgpu_status ybgpu_job_add_input_sst(ybgpu_job* job, const uint8_t* meta_file, uint64_t meta_file_len,
                                     const uint8_t* data_file, uint64_t data_file_len, uint64_t hybrid_time_filter) {
  if (!job) return YBGPU_INVALID_ARGUMENT;
  ybgpu::host::SstMeta m;
  std::string err = ybgpu::host::ParseSplitSstMeta(meta_file, meta_file_len, &m);
  if (!err.empty()) return JobFail(job, YBGPU_CORRUPTION, err);
  std::vector<ybgpu_block_handle> h(m.data_blocks.size());
  for (size_t i = 0; i < h.size(); i++) { h[i].offset = m.data_blocks[i].offset; h[i].size = m.data_blocks[i].size; }
  return ybgpu_job_add_input(job, data_file, data_file_len, h.data(), h.size(), m.key_encoding, hybrid_time_filter);
}

ybgpu_status ybgpu_job_run(ybgpu_job* job, const volatile int32_t* shutting_down) {
  if (!job) return YBGPU_INVALID_ARGUMENT;
  return Sync(job, job->engine->Run(shutting_down));
}

ybgpu_status ybgpu_job_verify_output(ybgpu_job* job, ybgpu_output_check* result) {
  if (!job || !result) return YBGPU_INVALID_ARGUMENT;
  return Sync(job, job->engine->VerifyOutput(result));
}

ybgpu_status ybgpu_sst_verify_device(int32_t device, const uint8_t* meta, uint64_t meta_len, const uint8_t* data, uint64_t data_len,
                                     ybgpu_output_check* result) {
  if (!meta || (!data && data_len) || !result) { g_last_error = "null argument"; return YBGPU_INVALID_ARGUMENT; }
  ybgpu::host::SstMeta m;
  std::string err = ybgpu::host::ParseSplitSstMeta(meta, meta_len, &m);
  if (!err.empty()) { g_last_error = err; return YBGPU_CORRUPTION; }
  std::vector<ybgpu_block_handle> h(m.data_blocks.size());
  for (size_t i = 0; i < h.size(); i++) { h[i].offset = m.data_blocks[i].offset; h[i].size = m.data_blocks[i].size; }
  ybgpu_job_options o;
  ybgpu_job_options_init(&o);
  o.device = device;
  o.cuda_stream = YBGPU_STREAM_PRIVATE;
  Engine e(o);
  ybgpu_status s = e.Init();
  if (s == YBGPU_OK) s = e.VerifySst(data, data_len, h.data(), h.size(), m.key_encoding, result);
  if (s != YBGPU_OK) g_last_error = e.error();
  return s;
}

ybgpu_status ybgpu_job_get_stats(const ybgpu_job* job, ybgpu_job_stats* stats) {
  if (!job || !stats) return YBGPU_INVALID_ARGUMENT;
  *stats = const_cast<ybgpu_job*>(job)->engine->stats();
  stats->num_output_data_blocks = job->num_blocks;
  stats->output_data_file_size = job->data_len;
  stats->output_meta_file_size = job->meta_file.size();
  return YBGPU_OK;
}

ybgpu_status ybgpu_job_kv_stream_sizes(const ybgpu_job* job, uint64_t* n, uint64_t* kb, uint64_t* vb) {
  if (!job) return YBGPU_INVALID_ARGUMENT;
  return Sync(const_cast<ybgpu_job*>(job), job->engine->KvStreamSizes(n, kb, vb));
}

ybgpu_status ybgpu_job_fetch_kv_stream(ybgpu_job* job, uint8_t* keys, uint64_t* koff, uint8_t* vals, uint64_t* voff) {
  if (!job) return YBGPU_INVALID_ARGUMENT;
  return Sync(job, job->engine->FetchKvStream(keys, koff, vals, voff));
}

static ybgpu_status EnsureHostKv(ybgpu_job* job) {
  if (job->have_kv) return YBGPU_OK;
  uint64_t n, kb, vb;
  ybgpu_status s = Sync(job, job->engine->KvStreamSizes(&n, &kb, &vb));
  if (s != YBGPU_OK) return s;
  job->keys.resize(kb + 1); job->vals.resize(vb + 1); job->koff.resize(n + 1); job->voff.resize(n + 1);
  s = Sync(job, job->engine->FetchKvStream(job->keys.data(), job->koff.data(), job->vals.data(), job->voff.data()));
  if (s == YBGPU_OK) job->have_kv = true;
  return s;
}

ybgpu_status ybgpu_job_emit_kv_stream(ybgpu_job* job, ybgpu_emit_fn emit, void* ctx) {
  if (!job || !emit) return YBGPU_INVALID_ARGUMENT;
  ybgpu_status s = EnsureHostKv(job);
  if (s != YBGPU_OK) return s;
  const uint64_t n = job->koff.size() - 1;
  for (uint64_t i = 0; i < n; i++) {
    int rc = emit(ctx, job->keys.data() + job->koff[i], job->koff[i + 1] - job->koff[i],
                  job->vals.data() + job->voff[i], job->voff[i + 1] - job->voff[i]);
    if (rc != 0) return JobFail(job, static_cast<ybgpu_status>(rc), "emit callback failed");
  }
  return YBGPU_OK;
}

// Output SST: the data file comes finished from the GPU (K5); the host writes the metadata file
// from per-block boundary keys and handles (index blocks, properties, metaindex, footer).
static ybgpu_status FetchSstParts(ybgpu_job* job) {
  ybgpu_job::SstParts& P = job->parts;
  if (P.fetched) return YBGPU_OK;
  Engine& e = *job->engine;
  ybgpu_status s = Sync(job, e.OutputInfo(&P.data_len, &P.nb, &P.stride));
  if (s != YBGPU_OK) return s;
  P.off.resize(static_cast<size_t>(P.nb) + 1);
  P.bnd.resize(static_cast<size_t>(P.nb) * 2 * P.stride);
  s = Sync(job, e.FetchOutput(nullptr, P.off.data(), P.bnd.data()));   // the data file itself goes straight to the caller
  if (s != YBGPU_OK) return s;
  if (P.nb && e.options().filter_policy != YBGPU_FILTER_NONE) {
    s = Sync(job, e.FilterInfo(&P.nfb, &P.fbytes, &P.fstride));
    if (s != YBGPU_OK) return s;
    P.filters.resize(static_cast<size_t>(P.nfb) * P.fbytes); P.fkeys.resize(static_cast<size_t>(P.nfb) * 2 * P.fstride);
    P.ffirst.resize(P.nfb); P.bfirst.resize(P.nb);
    s = Sync(job, e.FetchFilter(P.filters.data(), P.fkeys.data(), P.ffirst.data(), P.bfirst.data()));
    if (s != YBGPU_OK) return s;
  }
  P.fetched = true;
  return YBGPU_OK;
}

static ybgpu_status EnsureSst(ybgpu_job* job) {
  if (job->have_sst) return YBGPU_OK;
  Engine& e = *job->engine;
  const bool trace = getenv("YBGPU_TRACE") != nullptr;
  auto t_prev = std::chrono::steady_clock::now();
  auto tick = [&](const char* what) {
    if (!trace) return;
    auto now = std::chrono::steady_clock::now();
    fprintf(stderr, "[ybgpu trace] sst/%-12s %8.3f ms (host wall)\n", what, std::chrono::duration<double, std::milli>(now - t_prev).count());
    t_prev = now;
  };
  ybgpu_status s = FetchSstParts(job);
  if (s != YBGPU_OK) return s;
  tick("fetch parts");
  ybgpu_job::SstParts& P = job->parts;
  const uint64_t data_len = P.data_len; const uint32_t nb = P.nb, stride = P.stride;
  const std::vector<uint64_t>& off = P.off; const std::vector<uint8_t>& bnd = P.bnd;
  try {
    job->data_len = data_len;
    if (nb) {   // the reference never opens an output file for an empty result (compaction_job.cc:156-160)
      const ybgpu_job_options& o = e.options();
      ybgpu::host::TableOptions t;
      t.block_size = o.block_size; t.block_restart_interval = o.block_restart_interval;
      t.block_size_deviation = o.block_size_deviation; t.index_block_size = o.index_block_size;
      t.min_keys_per_index_block = o.min_keys_per_index_block; t.key_encoding = o.output_key_encoding;
      t.filter_policy = o.filter_policy; if (o.filter_block_size) t.filter_block_size = o.filter_block_size; t.compression = o.output_compression;
      ybgpu::host::MetaFileWriter w(t);
      // Filter blocks come finished from the GPU too. In the metadata file they are interleaved with
      // the index blocks in the order BlockBasedTableBuilder::Add produces them: filter block f is
      // written when the first key of block f+1 is added, i.e. at output entry first_entry[f+1], after
      // a data block cut at the same entry (block_based_table_builder.cc:508-528).
      const uint32_t nfb = P.nfb, fbytes = P.fbytes, fstride = P.fstride;
      const std::vector<uint8_t>& filters = P.filters; const std::vector<uint8_t>& fkeys = P.fkeys;
      const std::vector<uint32_t>& ffirst = P.ffirst; const std::vector<uint32_t>& bfirst = P.bfirst;
      uint32_t f = 0;
      std::string flast;
      auto flush_filter = [&](bool has_next) {
        const uint8_t* lk = fkeys.data() + static_cast<size_t>(2 * f + 1) * fstride;       // last key of block f
        flast.assign(reinterpret_cast<const char*>(lk + 2), lk[0] | (lk[1] << 8));
        const uint8_t* nk = has_next ? fkeys.data() + static_cast<size_t>(2 * (f + 1)) * fstride : nullptr;   // first key of block f+1
        w.AddFilterBlock(filters.data() + static_cast<size_t>(f) * fbytes, fbytes, &flast, nk ? nk + 2 : nullptr, nk ? (nk[0] | (nk[1] << 8)) : 0, has_next);
        f++;
      };
      std::string last;
      for (uint32_t b = 0; b < nb; b++) {
        // data block b is cut when entry bfirst[b+1] arrives; filter flushes of earlier entries come first
        // (the last data block is cut by Finish(), after every Add — hence after every such flush)
        while (nfb && f + 1 < nfb && (b + 1 >= nb || ffirst[f + 1] < bfirst[b + 1])) flush_filter(true);
        const uint8_t* lk = bnd.data() + static_cast<size_t>(2 * b) * stride;
        const uint8_t* nk = lk + stride;
        const size_t ll = lk[0] | (lk[1] << 8), nl = nk[0] | (nk[1] << 8);
        last.assign(reinterpret_cast<const char*>(lk + 2), ll);
        ybgpu::host::Handle h; h.offset = off[b]; h.size = off[b + 1] - off[b] - 5;
        w.AddDataBlock(&last, nk + 2, nl, b + 1 < nb, h);
      }
      if (nfb) flush_filter(false);                       // Finish(): the final filter block
      const ybgpu_job_stats& st = e.stats();
      ybgpu::host::MetaProps mp;
      mp.raw_key_size = st.total_output_raw_key_bytes; mp.raw_value_size = st.total_output_raw_value_bytes;
      mp.data_size = data_len; mp.num_entries = st.num_output_records; mp.num_data_blocks = nb;
      mp.deleted_keys = e.kept_deletions();
      tick("index+filter");
      w.Finish(mp);
      job->meta_file = w.meta_file();
      tick("finish");
    }
    job->num_blocks = nb;
    job->have_sst = true;
  } catch (const std::exception& ex) {
    return JobFail(job, YBGPU_NOT_SUPPORTED, ex.what());
  }
  return YBGPU_OK;
}

ybgpu_status ybgpu_job_output_sizes(const ybgpu_job* job, uint64_t* data_len, uint64_t* meta_len) {
  if (!job) return YBGPU_INVALID_ARGUMENT;
  ybgpu_status s = EnsureSst(const_cast<ybgpu_job*>(job));
  if (s != YBGPU_OK) return s;
  *data_len = job->data_len; *meta_len = job->meta_file.size();
  return YBGPU_OK;
}

ybgpu_status ybgpu_job_fetch_output(ybgpu_job* job, uint8_t* data_file, uint64_t data_cap, uint8_t* meta_file, uint64_t meta_cap) {
  if (!job) return YBGPU_INVALID_ARGUMENT;
  // The data file goes D2H straight into the caller's buffer on a copy stream; the host builds the
  // metadata file (index blocks, filter index, properties) while that DMA runs.
  uint64_t data_len = 0; uint32_t nb = 0, stride = 0;
  ybgpu_status s = Sync(job, job->engine->OutputInfo(&data_len, &nb, &stride));
  if (s != YBGPU_OK) return s;
  if (data_cap < data_len) return JobFail(job, YBGPU_INVALID_ARGUMENT, "output buffer too small");
  s = FetchSstParts(job);                 // small D2H copies first: they must not queue behind the data file
  if (s != YBGPU_OK) return s;
  s = Sync(job, job->engine->BeginFetchDataFile(data_file));
  if (s != YBGPU_OK) return s;
  s = EnsureSst(job);
  ybgpu_status s2 = Sync(job, job->engine->EndFetchDataFile());
  if (s != YBGPU_OK) return s;
  if (s2 != YBGPU_OK) return s2;
  if (meta_cap < job->meta_file.size()) return JobFail(job, YBGPU_INVALID_ARGUMENT, "output buffer too small");
  memcpy(meta_file, job->meta_file.data(), job->meta_file.size());
  return YBGPU_OK;
}

ybgpu_status ybgpu_job_output_boundaries(const ybgpu_job* job, uint8_t* smallest, uint64_t* smallest_len, uint8_t* largest, uint64_t* largest_len) {
  if (!job) return YBGPU_INVALID_ARGUMENT;
  ybgpu_job* j = const_cast<ybgpu_job*>(job);
  // two boundary-key records kept by the block encoder; the KV stream is not materialised for this
  uint64_t data_len = 0; uint32_t nb = 0, stride = 0;
  ybgpu_status s = Sync(j, j->engine->OutputInfo(&data_len, &nb, &stride));
  if (s != YBGPU_OK) return s;
  *smallest_len = 0; *largest_len = 0;
  if (nb == 0) return YBGPU_OK;
  std::vector<uint8_t> a(stride), b(stride);
  s = Sync(j, j->engine->FetchFileBoundaries(a.data(), b.data()));
  if (s != YBGPU_OK) return s;
  *smallest_len = a[0] | (a[1] << 8); *largest_len = b[0] | (b[1] << 8);
  memcpy(smallest, a.data() + 2, *smallest_len);
  memcpy(largest, b.data() + 2, *largest_len);
  return YBGPU_OK;
}

ybgpu_status ybgpu_job_output_user_values(ybgpu_job* job, ybgpu_user_value* smallest, ybgpu_user_value* largest, uint32_t cap, uint32_t* n) {
  if (!job || !smallest || !largest || !n) return YBGPU_INVALID_ARGUMENT;
  return Sync(job, job->engine->FetchUserValues(smallest, largest, cap, n));
}

ybgpu_status ybgpu_job_kv_stream_digest(ybgpu_job* job, uint64_t* digest) {
  if (!job) return YBGPU_INVALID_ARGUMENT;
  return Sync(job, job->engine->Digest(digest));
}

struct ybgpu_table_builder {
  std::unique_ptr<ybgpu::host::SplitSstWriter> w;
  bool finished = false;
};

ybgpu_status ybgpu_table_builder_create(const ybgpu_job_options* o, ybgpu_table_builder** b) {
  if (!o || !b) return YBGPU_INVALID_ARGUMENT;
  if (!ybgpu::host::OutputCompressionSupported(o->output_compression)) {
    g_last_error = ybgpu::host::UnsupportedOutputCompression(o->output_compression); return YBGPU_NOT_SUPPORTED;
  }
  try {
    ybgpu::host::TableOptions t;
    t.block_size = o->block_size; t.block_restart_interval = o->block_restart_interval;
    t.block_size_deviation = o->block_size_deviation; t.index_block_size = o->index_block_size;
    t.min_keys_per_index_block = o->min_keys_per_index_block; t.key_encoding = o->output_key_encoding;
    t.filter_policy = o->filter_policy; if (o->filter_block_size) t.filter_block_size = o->filter_block_size; t.compression = o->output_compression;
    std::unique_ptr<ybgpu_table_builder> tb(new ybgpu_table_builder);
    tb->w.reset(new ybgpu::host::SplitSstWriter(t));
    *b = tb.release();
    return YBGPU_OK;
  } catch (const std::exception& e) { g_last_error = e.what(); return YBGPU_NOT_SUPPORTED; }
}
ybgpu_status ybgpu_table_builder_add(ybgpu_table_builder* b, const uint8_t* key, uint64_t klen, const uint8_t* val, uint64_t vlen) {
  if (!b || b->finished || klen < 8) return YBGPU_INVALID_ARGUMENT;
  b->w->Add(key, klen, val, vlen);
  return YBGPU_OK;
}
ybgpu_status ybgpu_table_builder_finish(ybgpu_table_builder* b) {
  if (!b || b->finished) return YBGPU_INVALID_ARGUMENT;
  b->w->Finish(); b->finished = true;
  return YBGPU_OK;
}
uint64_t ybgpu_table_builder_num_entries(const ybgpu_table_builder* b) { return b->w->NumEntries(); }
uint64_t ybgpu_table_builder_total_file_size(const ybgpu_table_builder* b) { return b->w->TotalFileSize(); }
uint64_t ybgpu_table_builder_base_file_size(const ybgpu_table_builder* b) { return b->w->meta_file().size(); }
ybgpu_status ybgpu_table_builder_files(const ybgpu_table_builder* b, const uint8_t** d, uint64_t* dl, const uint8_t** m, uint64_t* ml) {
  if (!b || !b->finished) return YBGPU_ILLEGAL_STATE;
  *d = reinterpret_cast<const uint8_t*>(b->w->data_file().data()); *dl = b->w->data_file().size();
  *m = reinterpret_cast<const uint8_t*>(b->w->meta_file().data()); *ml = b->w->meta_file().size();
  return YBGPU_OK;
}
void ybgpu_table_builder_destroy(ybgpu_table_builder* b) { delete b; }

ybgpu_status ybgpu_sst_meta_handles(const uint8_t* meta, uint64_t len, ybgpu_block_handle* handles, uint64_t cap,
                                    uint64_t* n, int32_t* enc) {
  if (!meta || !n) return YBGPU_INVALID_ARGUMENT;
  ybgpu::host::SstMeta m;
  std::string err = ybgpu::host::ParseSplitSstMeta(meta, len, &m);
  if (!err.empty()) { g_last_error = err; return YBGPU_CORRUPTION; }
  *n = m.data_blocks.size();
  if (enc) *enc = m.key_encoding;
  if (handles) {
    if (cap < m.data_blocks.size()) return YBGPU_INVALID_ARGUMENT;
    for (size_t i = 0; i < m.data_blocks.size(); i++) { handles[i].offset = m.data_blocks[i].offset; handles[i].size = m.data_blocks[i].size; }
  }
  return YBGPU_OK;
}

ybgpu_status ybgpu_sst_meta_separators(const uint8_t* meta, uint64_t len, uint8_t* keys, uint64_t cap, uint64_t* offs,
                                       uint64_t* n, uint64_t* bytes) {
  if (!meta || !n || !bytes) return YBGPU_INVALID_ARGUMENT;
  ybgpu::host::SstMeta m;
  std::string err = ybgpu::host::ParseSplitSstMeta(meta, len, &m);
  if (!err.empty()) { g_last_error = err; return YBGPU_CORRUPTION; }
  uint64_t total = 0;
  for (auto& k : m.separators) total += k.size();
  *n = m.separators.size(); *bytes = total;
  if (keys && offs) {
    if (cap < total) return YBGPU_INVALID_ARGUMENT;
    uint64_t o = 0;
    for (size_t i = 0; i < m.separators.size(); i++) { offs[i] = o; memcpy(keys + o, m.separators[i].data(), m.separators[i].size()); o += m.separators[i].size(); }
    offs[m.separators.size()] = o;
  }
  return YBGPU_OK;
}

ybgpu_status ybgpu_sst_concat_meta(const ybgpu_job_options* o, const ybgpu_sst_piece* pieces, uint32_t n, uint8_t* meta_out,
                                   uint64_t meta_cap, uint64_t* meta_len) {
  if (!o || !pieces || !meta_len || n == 0) { g_last_error = "null argument"; return YBGPU_INVALID_ARGUMENT; }
  if (!meta_out) {
    // size bound: filter blocks are copied as they are; an index entry (key delta + handle, >= ~10 bytes)
    // grows by at most the 5 extra varint bytes of a rebased offset
    uint64_t total = 65536;
    for (uint32_t i = 0; i < n; i++) total += 2 * pieces[i].meta_file_len + 256;
    *meta_len = total;
    return YBGPU_OK;
  }
  ybgpu::host::TableOptions t;
  t.block_size = o->block_size; t.block_restart_interval = o->block_restart_interval;
  t.block_size_deviation = o->block_size_deviation; t.index_block_size = o->index_block_size;
  t.min_keys_per_index_block = o->min_keys_per_index_block; t.key_encoding = o->output_key_encoding;
  t.filter_policy = o->filter_policy; if (o->filter_block_size) t.filter_block_size = o->filter_block_size; t.compression = o->output_compression;
  std::vector<ybgpu::host::SstPiece> ps(n);
  for (uint32_t i = 0; i < n; i++) {
    ps[i].meta = pieces[i].meta_file; ps[i].meta_len = pieces[i].meta_file_len; ps[i].data_len = pieces[i].data_file_len;
    if (pieces[i].smallest_key) ps[i].smallest.assign(reinterpret_cast<const char*>(pieces[i].smallest_key), pieces[i].smallest_key_len);
    if (pieces[i].largest_key) ps[i].largest.assign(reinterpret_cast<const char*>(pieces[i].largest_key), pieces[i].largest_key_len);
  }
  std::string out;
  std::string err = ybgpu::host::ConcatSplitSstMeta(t, ps, &out);
  if (!err.empty()) { g_last_error = err; return YBGPU_INVALID_ARGUMENT; }
  *meta_len = out.size();
  if (out.size() > meta_cap) { g_last_error = "metadata buffer too small"; return YBGPU_INVALID_ARGUMENT; }
  memcpy(meta_out, out.data(), out.size());
  return YBGPU_OK;
}

}  // extern "C"

// Whether the first bytes of a block labelled LZ4 / LZ4HC can open a stream the engine decodes: a varint32 preamble
// below k_snappy_sizes' 2^30 limit, then a raw LZ4 block, which is exactly one byte (an empty token) when the announced
// length is 0 and longer otherwise (a non-empty output needs a token and its literals). Reads at most 5 bytes.
static bool Lz4PreambleFits(const uint8_t* p, uint64_t n) {
  uint64_t u = 0;
  for (uint64_t i = 0; i < 5 && i < n; i++) {
    u |= static_cast<uint64_t>(p[i] & 127) << (7 * i);
    if (!(p[i] & 128)) {
      const uint64_t body = n - i - 1;
      return u < (1u << 30) && body >= 1 && (u == 0) == (body == 1);
    }
  }
  return false;
}

extern "C" {

ybgpu_status ybgpu_sst_check_supported(const uint8_t* meta, uint64_t meta_len, const uint8_t* data, uint64_t data_len, uint64_t counts[8]) {
  if (!meta || (!data && data_len)) { g_last_error = "null argument"; return YBGPU_INVALID_ARGUMENT; }
  ybgpu::host::SstMeta m;
  std::string err = ybgpu::host::ParseSplitSstMeta(meta, meta_len, &m);
  if (!err.empty()) { g_last_error = err; return YBGPU_CORRUPTION; }
  uint64_t local[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  uint64_t lz4_unfit = 0;                                   // blocks labelled LZ4 whose first bytes open no LZ4 stream
  for (const ybgpu::host::Handle& h : m.data_blocks) {
    if (h.offset > data_len || h.size > data_len - h.offset || data_len - h.offset - h.size < 5) {
      g_last_error = "a data block handle points outside the data file"; return YBGPU_CORRUPTION;
    }
    const uint8_t type = data[h.offset + h.size];
    if (type > 7) { g_last_error = "unknown block compression type " + std::to_string(type); return YBGPU_CORRUPTION; }
    local[type]++;
    if ((type == 4 || type == 5) && !Lz4PreambleFits(data + h.offset, h.size)) lz4_unfit++;
  }
  if (counts) memcpy(counts, local, sizeof(local));
  if (m.key_encoding != YBGPU_KEY_ENCODING_SHARED_PREFIX && m.key_encoding != YBGPU_KEY_ENCODING_THREE_SHARED_PARTS) {
    g_last_error = "data block key-value encoding format " + std::to_string(m.key_encoding) + " is not decoded by the engine"; return YBGPU_NOT_SUPPORTED;
  }
  for (int t = 2; t < 8; t++)
    if (local[t] && t != 4 && t != 5) {
      static const char* const kNames[8] = {"none", "snappy", "zlib", "bzip2", "lz4", "lz4hc", "xpress", "zstd"};
      g_last_error = std::to_string(local[t]) + " data blocks are stored with " + kNames[t] +
                     " compression: only raw, Snappy and LZ4 (LZ4HC) blocks are decoded on the GPU";
      return YBGPU_NOT_SUPPORTED;
    }
  if (lz4_unfit) {
    g_last_error = std::to_string(lz4_unfit) + " data blocks labelled LZ4 do not start with an LZ4 length preamble the engine decodes";
    return YBGPU_NOT_SUPPORTED;
  }
  return YBGPU_OK;
}

ybgpu_status ybgpu_sst_uncompressed_bytes(const uint8_t* meta, uint64_t meta_len, const uint8_t* data, uint64_t data_len,
                                         uint64_t* image_bytes, uint64_t* compressed_blocks) {
  if (!meta || (!data && data_len) || !image_bytes || !compressed_blocks) { g_last_error = "null argument"; return YBGPU_INVALID_ARGUMENT; }
  ybgpu::host::SstMeta m;
  std::string err = ybgpu::host::ParseSplitSstMeta(meta, meta_len, &m);
  if (!err.empty()) { g_last_error = err; return YBGPU_CORRUPTION; }
  for (const ybgpu::host::Handle& h : m.data_blocks)
    if (h.offset > data_len || h.size > data_len - h.offset || data_len - h.offset - h.size < 5) {
      g_last_error = "a data block handle points outside the data file"; return YBGPU_CORRUPTION;
    }
  *image_bytes = ybgpu::host::UncompressedImageBytes(data, m.data_blocks.data(), m.data_blocks.size(), compressed_blocks);
  return YBGPU_OK;
}

ybgpu_status ybgpu_sst_verify_blocks(const uint8_t* meta, uint64_t meta_len, const uint8_t* data, uint64_t data_len, uint32_t stride,
                                     uint64_t* checked, uint64_t* bad) {
  if (!meta || !data || !checked || !bad) return YBGPU_INVALID_ARGUMENT;
  ybgpu::host::SstMeta m;
  std::string err = ybgpu::host::ParseSplitSstMeta(meta, meta_len, &m);
  if (!err.empty()) { g_last_error = err; return YBGPU_CORRUPTION; }
  if (stride == 0) stride = 1;
  *checked = 0; *bad = 0;
  for (size_t i = 0; i < m.data_blocks.size(); i += stride) {
    const ybgpu::host::Handle& h = m.data_blocks[i];
    (*checked)++;
    if (h.offset + h.size + 5 > data_len) { (*bad)++; continue; }
    const uint8_t* p = data + h.offset;
    uint32_t stored; memcpy(&stored, p + h.size + 1, 4);
    const uint8_t type = p[h.size];                        // none, Snappy, LZ4, LZ4HC: the checksum covers the stored bytes
    if ((type > 1 && type != 4 && type != 5) || ybgpu::host::Crc32cMask(ybgpu::host::Crc32c(p, h.size + 1)) != stored) (*bad)++;
  }
  if (*bad) { g_last_error = "block checksum mismatch"; return YBGPU_CORRUPTION; }
  return YBGPU_OK;
}

int32_t ybgpu_device_count(void);   // engine.cu
const char* ybgpu_version(void) { return "ybgpu-compaction 0.1 (sm_90a)"; }

}  // extern "C"
