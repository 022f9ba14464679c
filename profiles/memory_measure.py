"""Device memory of a compaction job per input shape, and what a budget costs a pipelined one, in one run on one card.
Usage: python profiles/memory_measure.py [--rows 2000000] [--out DIR]

Per shape (the bench generator shape; MVCC-heavy; Snappy and LZ4 inputs; Snappy and LZ4 outputs; bloom filters;
verify_output; KV inputs; colocated tables): input bytes (the data files, or the KV streams' key + value bytes),
ybgpu_job_stats::device_bytes_peak, the default pool's cudaMemPoolAttrUsedMemHigh delta over the job, and peak / input.
Then the end-to-end time of compact_files_one_table (host -> device -> host, one table out, max_in_flight 3) over the
bench shape with no budget and with budgets of 1x, 1/2x and 1/4x of the single job's unbudgeted peak (max_subcompactions
0: planned from the budget), with the ranges it ran and its total device_bytes_peak. Prints the card and its power limit
first; writes the same lines to DIR/memory_measure.txt when --out is given."""
import argparse
import ctypes as C
import importlib
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]
pkg = importlib.import_module("yugabyte-db_b200")
if pkg.device_count() < 1:
    raise SystemExit("memory_measure.py needs a CUDA device")
import oracle_py as o  # noqa: E402
import lz4_util as z  # noqa: E402
import workloads as w  # noqa: E402
from test_gpu_parity import _phrase_runs  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=2000000)
ap.add_argument("--out", default=None)
args = ap.parse_args()
lines = []


def emit(s):
    print(s, flush=True)
    lines.append(s)


emit(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                    capture_output=True, text=True).stdout.strip())

pkg.lib()
rt = C.CDLL("libcudart.so.12")
pool = C.c_void_p()
assert rt.cudaDeviceGetDefaultMemPool(C.byref(pool), 0) == 0


def pool_attr(attr):
    v = C.c_uint64()
    assert rt.cudaMemPoolGetAttribute(pool, attr, C.byref(v)) == 0
    return v.value


def reset_high():
    rt.cudaDeviceSynchronize()
    zero = C.c_uint64(0)
    assert rt.cudaMemPoolSetAttribute(pool, 8, C.byref(zero)) == 0
    return pool_attr(7)


def measure(name, tables=None, kvs=None, verify=False, **kw):
    base = reset_high()
    job = pkg.GpuCompactionJob(**kw)
    if tables is not None:
        for m, d in tables:
            job.add_input_sst(m, d)
        in_bytes = sum(int(d.size) for _, d in tables)
    else:
        for r in kvs:
            job.add_input_kv(r)
        in_bytes = sum(len(k) + len(v) for r in kvs for k, v in r)
    job.run()
    if verify:
        job.verify_output()
    rt.cudaDeviceSynchronize()
    peak = job.stats().device_bytes_peak
    delta = pool_attr(8) - base
    job.close()
    emit("%-16s input %12d B  device_bytes_peak %12d B  pool UsedMemHigh delta %12d B  (+%d)  peak/input %.2f" % (
        name, in_bytes, peak, delta, delta - peak, peak / max(1, in_bytes)))
    return peak


bench = pkg.generate_ssts(pkg.GenConfig(seed=2, num_rows=args.rows, cols=1, versions=1, num_files=8, value_len=256), max_threads=8)
bench_v = [(s.meta_view(), s.data_view()) for s in bench]
mvcc = pkg.generate_ssts(pkg.GenConfig(seed=3, num_rows=args.rows // 8, cols=2, versions=8, num_files=4, value_len=64,
                                       tombstone_per_1024=100), max_threads=8)
mvcc_v = [(s.meta_view(), s.data_view()) for s in mvcc]
cut = o.ht_from_micros(1790000000 * 1000000 + 4000)
phr = _phrase_runs(5, 3, max(1000, args.rows // 200))
snap = [o.Sst.build(r, o.TableOptions(block_size=32768, compression=1)) for r in phr]
lz4 = [z.host_lz4_table(pkg, r, block_size=32768) for r in phr]
raw_phr = [o.Sst.build(r, o.TableOptions(block_size=32768)) for r in phr]
cot = [o.Sst.build(r, o.TableOptions(block_size=4096)) for r in w.random_cotable_runs(7, n_runs=4, n_tables=50, rows_per_table=200) if r]
small = [s.read_all() for s in o.Sst.generate_all(o.GenConfig(seed=9, num_rows=50000, cols=2, versions=3, num_files=3, value_len=100),
                                                   o.TableOptions(block_size=4096))]
views = lambda ts: [(t.meta_view(), t.data_view()) for t in ts]  # noqa: E731

emit("-- device memory per shape")
bench_peak = measure("bench", bench_v, filter_policy=1)
measure("mvcc_heavy", mvcc_v, cutoff_ht=cut)
measure("snappy_in", views(snap))
measure("lz4_in", views(lz4))
measure("snappy_out", views(raw_phr), output_compression=1)
measure("lz4_out", views(raw_phr), output_compression=4)
measure("filters", mvcc_v, cutoff_ht=cut, filter_policy=1)
measure("verify_output", views(raw_phr), verify=True, output_compression=1)
measure("kv_inputs", kvs=small, retention=False)
measure("colocated", views(cot), block_size=4096)

emit("-- compact_files_one_table over the bench shape (filters on, max_in_flight 3), budget relative to the single job's peak %d B" % bench_peak)
for label, budget, max_sub in (("none, 8 ranges", 0, 8), ("1x", bench_peak, 0), ("1/2x", bench_peak // 2, 0), ("1/4x", bench_peak // 4, 0)):
    best = None
    for rep in range(3):
        rt.cudaDeviceSynchronize()
        t0 = time.perf_counter()
        data, meta, res, total = pkg.compact_files_one_table(bench_v, max_subcompactions=max_sub, max_in_flight=3,
                                                             device_memory_budget=budget, filter_policy=1)
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    emit("budget %-14s %7.3f s (best of 3)  ranges %4d  total device_bytes_peak %12d B  data %d B" % (
        label, best, res.num_ranges, total.device_bytes_peak, res.data_len))

if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "memory_measure.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")
