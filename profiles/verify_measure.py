"""What the device-side output check (ybgpu_job_verify_output) costs next to the job it checks, in one run on one card.
Usage: python profiles/verify_measure.py [--rows 40000000] [--steps 5] [--warmup 2]

The bench shape (8 files, 256-byte values, 32 KB blocks, DocKeyV3 bloom filters, input checksums verified), input files
resident in HBM, for output compression none / Snappy / LZ4: per timed step the job's kernel time (stats.gpu_seconds) and
the check's device time (CUDA events on the job's stream, ybgpu_output_check.gpu_seconds), the bytes the check reads
(computed by the engine from the table's sizes: stored table + uncompressed image + the values and key records it compares
with) and the rate that gives. For comparison, the host check the adapter's CheckOutputFile(paranoid = true) makes
(ybgpu_sst_verify_blocks, every block, one host thread) is timed once per compression on the fetched table. Prints the
card and its power limit first."""
import argparse
import importlib
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]
pkg = importlib.import_module("yugabyte-db_b200")
if pkg.device_count() < 1:
    raise SystemExit("verify_measure.py needs a CUDA device")

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=40000000)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=2)
args = ap.parse_args()

print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())

cfg = pkg.GenConfig(seed=2, num_rows=args.rows, cols=1, versions=1, num_files=8, value_len=256)
ssts = pkg.generate_ssts(cfg, max_threads=8)
handles = [pkg.sst_block_handles(s.meta_view())[:2] for s in ssts]
dev_files = []
for s in ssts:
    v = s.data_view()
    t = torch.zeros(v.size + 64, dtype=torch.uint8, device="cuda")
    t[16:16 + v.size].copy_(torch.from_numpy(v))
    dev_files.append(t)
torch.cuda.synchronize()
stream = torch.cuda.current_stream().cuda_stream
print("inputs: %d entries, %.2f GB of data files" % (sum(s.num_entries for s in ssts), sum(s.data_view().size for s in ssts) / 1e9))

for comp, name in ((0, "none"), (1, "snappy"), (4, "lz4")):
    rows = []
    for step in range(args.warmup + args.steps):
        job = pkg.GpuCompactionJob(verify_checksums=True, cuda_stream=stream, filter_policy=1, output_compression=comp)
        for t, s, (off, sz) in zip(dev_files, ssts, handles):
            job.add_input_device(t.data_ptr() + 16, s.data_view().size, off, sz)
        st = job.run()
        chk = job.verify_output()
        assert job.stats().path_flags & pkg.PATH_OUTPUT_VERIFIED
        if step >= args.warmup:
            rows.append((st.gpu_seconds, chk.gpu_seconds, chk.bytes_read, chk.blocks_checked, chk.blocks_compressed, chk.entries_parsed))
        if step == args.warmup + args.steps - 1:
            data, meta = job.fetch_output()
            t0 = time.perf_counter()
            checked, bad = pkg.sst_verify_blocks(meta, data, 1)
            host_s = time.perf_counter() - t0
            table_bytes = data.size
        job.close()
    job_ms = np.array([r[0] for r in rows]) * 1e3
    chk_ms = np.array([r[1] for r in rows]) * 1e3
    print("output compression %-6s: %d blocks (%d stored compressed), %d entries, table %.2f GB" % (name, rows[-1][3], rows[-1][4], rows[-1][5], table_bytes / 1e9))
    print("  job kernels      %s ms (median %.2f)" % (" ".join("%.2f" % x for x in job_ms), np.median(job_ms)))
    print("  device check     %s ms (median %.2f): %.2f GB read, %.0f GB/s, %.0f %% of the job's kernel time"
          % (" ".join("%.2f" % x for x in chk_ms), np.median(chk_ms), rows[-1][2] / 1e9, rows[-1][2] / np.median(chk_ms) / 1e6,
             100 * np.median(chk_ms) / np.median(job_ms)))
    print("  host check (every block's checksum, one thread, after the copy): %.0f ms, %d blocks, %d bad" % (host_s * 1e3, checked, bad))
