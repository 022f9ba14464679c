#!/usr/bin/env python
"""profiles/e2e_sweep.py — explores the end-to-end (host files in, host files out) arm of bench.py on a GPU
box: one set of config-2 inputs, then ybgpu_compact_files_one_table under several settings (number of key ranges,
ranges in flight, copy slots = ranges whose inputs are in transit / that copy out at once). Prints one JSON line per setting;
`--trace` adds the per-range timeline of one step (YBGPU_SUB_TRACE) on stderr. Not a bench value source:
bench.py measures the committed defaults.

    python profiles/e2e_sweep.py --rows 40000000 > e2e_sweep.jsonl 2> e2e_sweep.err
"""
import argparse
import importlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--trace", action="store_true")
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--grid", default="", help="settings to run instead of the built-in grid: 'ranges,in_flight,h2d_slots,d2h_slots;...'")
    args = ap.parse_args()
    import torch
    pkg = importlib.import_module("yugabyte-db_b200")
    torch.cuda.set_device(0)
    cfg = pkg.GenConfig(seed=2, num_rows=args.rows, cols=1, versions=1, num_files=8, value_len=256, hash_rows_total=args.rows)
    ssts = pkg.generate_ssts(cfg, max_threads=8)
    in_bytes = sum(s.raw_bytes for s in ssts)
    file_bytes = sum(s.data_view().size for s in ssts)
    cudart = torch.cuda.cudart()
    for s in ssts:
        v = s.data_view()
        assert int(cudart.cudaHostRegister(v.ctypes.data, v.size, 0)) == 0
    out_data = torch.empty(file_bytes + (64 << 20), dtype=torch.uint8, pin_memory=True).numpy()
    out_meta = torch.empty(max(64 << 20, file_bytes // 100), dtype=torch.uint8, pin_memory=True).numpy()
    files = [(s.meta_view(), s.data_view()) for s in ssts]

    def run(subs, inflight, h2d_slots, d2h_slots, steps, one_table=True, chunk_mb=32, zc=1):
        os.environ["YBGPU_COPY_CHUNK_MB"] = str(chunk_mb)
        os.environ["YBGPU_ZC_STATUS"] = str(zc)
        os.environ["YBGPU_H2D_SLOTS"] = str(h2d_slots)
        os.environ["YBGPU_D2H_SLOTS"] = str(d2h_slots)
        best, tot = None, 0.0
        for i in range(steps + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if one_table:
                _, _, res, total = pkg.compact_files_one_table(files, max_subcompactions=subs, max_in_flight=inflight, data_out=out_data,
                                                               meta_out=out_meta, filter_policy=1, verify_checksums=True)
                n_ranges = res.num_ranges
            else:
                r = pkg.compact_files(files, max_subcompactions=subs, max_in_flight=inflight, data_arena=out_data,
                                      meta_arena=out_meta, filter_policy=1, verify_checksums=True)
                total, n_ranges = r.total, len(r.outputs)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            assert total.num_input_records == args.rows
            if i:
                tot += dt
                best = dt if best is None else min(best, dt)
        print(json.dumps({"one_table": one_table, "subcompactions": subs, "in_flight": inflight, "h2d_slots": h2d_slots, "d2h_slots": d2h_slots,
                          "chunk_mb": chunk_mb, "zero_copy_status": zc, "ranges": n_ranges, "ms_per_step": round(tot / steps * 1e3, 1),
                          "best_ms": round(best * 1e3, 1), "gb_per_s": round(in_bytes * steps / tot / 1e9, 2),
                          "gpu_ms_sum": round(total.gpu_seconds * 1e3, 1)}), flush=True)

    # (ranges, in flight, ranges with inputs in transit, ranges copying out); slots 0 = ungated (round-1 behaviour)
    grid = [(32, 6, 0, 0), (32, 6, 2, 2), (32, 8, 2, 2), (32, 12, 2, 2), (32, 12, 1, 1), (32, 12, 2, 1), (32, 12, 1, 2), (32, 12, 3, 3),
            (64, 12, 2, 2), (64, 16, 2, 2), (16, 8, 2, 2), (48, 12, 2, 2)]
    if args.quick:
        grid = grid[:5]
    if args.grid:
        grid = [tuple(int(x) for x in g.split(',')) for g in args.grid.split(';')]
    for g in grid:
        run(*g, steps=args.steps)
    if args.trace:
        os.environ["YBGPU_SUB_TRACE"] = "1"
        run(32, 12, 2, 2, steps=1)


if __name__ == "__main__":
    main()
