"""Where the encode phase's time goes outside the block assembler: every kernel between k_merge_filter and the end of
the job, one row per kernel name, in one run on one card.
Usage: python profiles/plan_measure.py [--rows 40000000] [--steps 3] [--warmup 2] [--trace-dir DIR]

The bench shape (bench.py's generator call: seed 2, 8 files, 256-byte values; DocKeyV3 bloom filters, input checksums
verified), input files resident in HBM. After the warm-up, --steps jobs run under torch.profiler with CUDA activities
(CUPTI sees the library's kernels too; Nsight is not needed). A one-element torch kernel on the job's stream marks the
end of every job. Per kernel name (memsets and copies on the stream are rows too), per job: launches, total and mean
device time, and the idle time on the stream in front of it (start minus the end of the previous activity, which is
launch latency or a host round trip). Below the table: the span from the end of k_merge_filter to the end of the last
kernel, the sum of the kernels in it, and their difference. Prints the card and its power limit first; profiling slows
the host, so the gaps are upper bounds and end-to-end figures come from bench.py."""
import argparse
import collections
import importlib
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]
pkg = importlib.import_module("yugabyte-db_b200")

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=40000000)
ap.add_argument("--steps", type=int, default=3)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--trace-dir", default=None, help="where the chrome trace is written (default: a temporary directory)")
args = ap.parse_args()

cfg = pkg.GenConfig(seed=2, num_rows=args.rows, cols=1, versions=1, num_files=8, value_len=256)
ssts = pkg.generate_ssts(cfg, max_threads=8)
handles = [pkg.sst_block_handles(s.meta_view())[:2] for s in ssts]
print("inputs: %d entries, %.2f GB of data files" % (sum(s.num_entries for s in ssts), sum(s.data_view().size for s in ssts) / 1e9))
if not torch.cuda.is_available() or pkg.device_count() < 1:
    raise SystemExit("plan_measure.py needs a CUDA device: kernel times cannot be taken without one")

print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())

dev_files = []
for s in ssts:
    v = s.data_view()
    t = torch.zeros(v.size + 64, dtype=torch.uint8, device="cuda")
    t[16:16 + v.size].copy_(torch.from_numpy(v))
    dev_files.append(t)
torch.cuda.synchronize()
stream = torch.cuda.current_stream().cuda_stream
marker = torch.zeros(1, dtype=torch.int32, device="cuda")


def one_job():
    job = pkg.GpuCompactionJob(verify_checksums=True, cuda_stream=stream, filter_policy=1)
    for t, s, (off, sz) in zip(dev_files, ssts, handles):
        job.add_input_device(t.data_ptr() + 16, s.data_view().size, off, sz)
    st = job.run()
    marker.add_(1)                                  # end-of-job mark on the job's stream
    torch.cuda.synchronize()
    job.close()
    return st


for _ in range(args.warmup):
    st = one_job()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
    stats = [one_job() for _ in range(args.steps)]
trace_dir = args.trace_dir or tempfile.mkdtemp(prefix="plan_measure_")
os.makedirs(trace_dir, exist_ok=True)
trace_path = os.path.join(trace_dir, "plan_measure_trace.json")
prof.export_chrome_trace(trace_path)

with open(trace_path) as f:
    events = json.load(f)["traceEvents"]
acts = sorted((e for e in events if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")), key=lambda e: e["ts"])


def short(name):
    name = name.split("(")[0]
    return name.split("::")[-1] if name.startswith("ybgpu::") or "ybgpu::" in name else name


# split into jobs at the marker kernel (the only torch elementwise kernel in the window)
jobs, cur = [], []
for e in acts:
    if e["cat"] == "kernel" and "elementwise" in e["name"]:
        jobs.append(cur)
        cur = []
    else:
        cur.append(e)
if len(jobs) != args.steps:
    raise SystemExit("expected %d jobs in the trace, found %d" % (args.steps, len(jobs)))

rows = collections.OrderedDict()
spans, sums = [], []
for job in jobs:
    idx = [i for i, e in enumerate(job) if "k_merge_filter" in e["name"]]
    if len(idx) != 1:
        raise SystemExit("a job without exactly one k_merge_filter launch")
    m = idx[0]
    prev_end = job[m]["ts"] + job[m]["dur"]
    phase_start = prev_end
    total = 0.0
    for e in job[m + 1:]:
        r = rows.setdefault(short(e["name"]) if e["cat"] == "kernel" else e["cat"] + " " + e["name"].split("(")[0].strip(), [0, 0.0, 0.0])
        r[0] += 1; r[1] += e["dur"]; r[2] += max(0.0, e["ts"] - prev_end)
        total += e["dur"]
        prev_end = max(prev_end, e["ts"] + e["dur"])
    spans.append(prev_end - phase_start)
    sums.append(total)

nj = len(jobs)
print("\nkernels after k_merge_filter, per job (mean of %d profiled jobs; %d entries out, %d launches per job)" % (
    nj, stats[-1].num_output_records, stats[-1].gpu_kernel_launches))
print("| activity | launches | total ms | mean us | idle in front, ms |")
print("|---|---|---|---|---|")
for name, (cnt, dur, gap) in rows.items():
    print("| `%s` | %.4g | %.3f | %.1f | %.3f |" % (name, cnt / nj, dur / nj / 1e3, dur / cnt, gap / nj / 1e3))
print("\nspan from the end of k_merge_filter to the end of the last kernel: %s ms" % " ".join("%.3f" % (x / 1e3) for x in spans))
print("sum of the activities in it:                                       %s ms" % " ".join("%.3f" % (x / 1e3) for x in sums))
print("difference (launch gaps and host round trips, profiler attached):   %s ms" % " ".join("%.3f" % ((a - b) / 1e3) for a, b in zip(spans, sums)))
print("CUDA-event times of the last job (no profiler influence on these): phases %s ms, block assembler %.3f ms" % (
    " ".join("%.3f" % (x * 1e3) for x in stats[-1].phase_seconds[:5]), stats[-1].phase_seconds[5] * 1e3))
