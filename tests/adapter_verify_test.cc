// Compiled by tests/test_gpu_verify.py: the C++ adapter with Params::paranoid_file_checks (the device-side output check
// inside Run()). argv[1] = max_subcompactions, argv[2..] = pairs (base file, data file) of the input tables. Snappy
// output; prints "OK <entries parsed by the check> <output files>" or the failing status.
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iterator>
#include "../yugabyte-db_b200/csrc/adapter/gpu_compaction_job.h"

using namespace ybgpu_adapter;

static std::string ReadFile(const char* p) { std::ifstream f(p, std::ios::binary); return std::string(std::istreambuf_iterator<char>(f), {}); }

int main(int argc, char** argv) {
  if (argc < 4 || (argc - 2) % 2) { printf("usage\n"); return 2; }
  std::vector<std::string> keep;
  for (int i = 2; i < argc; i++) keep.push_back(ReadFile(argv[i]));
  std::vector<InputFile> inputs;
  for (size_t i = 0; i + 1 < keep.size(); i += 2) {
    InputFile f;
    f.base_file = Slice(keep[i]); f.data_file = Slice(keep[i + 1]);
    inputs.push_back(f);
  }
  GpuCompactionJob::Params p;
  p.block_size = 4096;
  p.output_compression = YBGPU_COMPRESSION_SNAPPY;
  p.max_subcompactions = static_cast<uint32_t>(atoi(argv[1]));
  p.paranoid_file_checks = true;
  GpuCompactionJob job(p);
  Status s = job.Prepare(inputs);
  if (s.ok()) s = job.Run();
  if (!s.ok()) { printf("%s\n", s.ToString().c_str()); return 1; }
  if (!(job.stats().path_flags & YBGPU_PATH_OUTPUT_VERIFIED)) { printf("output not verified\n"); return 1; }
  s = job.CheckOutputFile(true);                           // the host check of the copied bytes still passes
  if (!s.ok()) { printf("host check: %s\n", s.ToString().c_str()); return 1; }
  const unsigned long long parsed = p.max_subcompactions > 1 ? job.stats().num_output_records : job.output_check().entries_parsed;
  if (parsed != job.stats().num_output_records) { printf("the check parsed %llu of %llu entries\n", parsed, (unsigned long long)job.stats().num_output_records); return 1; }
  printf("OK %llu %zu\n", parsed, p.max_subcompactions > 1 ? job.outputs().size() : size_t(1));
  return 0;
}
