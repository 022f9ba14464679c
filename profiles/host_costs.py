#!/usr/bin/env python
"""profiles/host_costs.py — host-side (CPU-only) costs of the pieces around the GPU path that sit inside the
end-to-end timed region: the subcompaction planner (ybgpu_plan_subcompactions: parse every input's index,
pick row-aligned splitters) and the one-table assembly (ybgpu_sst_concat_meta). Inputs have the index size
of BASELINE config 2 (8 inputs, ~9.2e5 data blocks in total); data blocks are 4 KB here instead of 32 KB so
that the files stay small. Needs no GPU.

    python profiles/host_costs.py > host_costs.json
"""
import importlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]


def first_key(d):
    pos, vals = 0, []
    for _ in range(3):
        v = shift = 0
        while True:
            c = int(d[pos]); pos += 1
            v |= (c & 0x7f) << shift; shift += 7
            if not c & 0x80:
                break
        vals.append(v)
    return bytes(d[pos:pos + vals[1]])


def main():
    import numpy as np
    import oracle_py as o            # generator with bloom filter blocks (tooling only)
    pkg = importlib.import_module("yugabyte-db_b200")
    P, n = 8, 1_500_000
    pieces, files = [], []
    keep = []
    for i in range(P):
        cfg = o.GenConfig(seed=2, num_rows=n, cols=1, versions=1, num_files=1, value_len=256, row_offset=i * n, hash_rows_total=P * n)
        s = o.Sst.generate(cfg, 0, o.TableOptions(block_size=4096, filter_policy=1, filter_block_size=65536))
        meta, data = s.meta_view().copy(), s.data_view()
        pieces.append((meta, data.size, first_key(data), pkg.sst_last_key(meta, data)))
        files.append((meta, data))
        keep.append(s)
    blocks = sum(len(pkg.sst_block_handles(m)[0]) for m, _ in files)

    def best(fn, reps=5):
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
        return min(ts), sorted(ts)[len(ts) // 2]
    out = np.empty(2 * sum(len(p[0]) for p in pieces) + (1 << 20), np.uint8)
    plan = best(lambda: pkg.plan_subcompactions(files, 32))
    concat = best(lambda: pkg.sst_concat_meta(pieces, out=out, block_size=4096, filter_policy=1, filter_block_size=65536))
    print(json.dumps({
        "host_cores": os.cpu_count(), "inputs": P, "data_blocks_total": blocks,
        "meta_bytes_total": int(sum(len(p[0]) for p in pieces)),
        "plan_subcompactions_32_ranges_s": {"best": round(plan[0], 4), "median": round(plan[1], 4)},
        "sst_concat_meta_s": {"best": round(concat[0], 4), "median": round(concat[1], 4)},
        "note": "config 2 proper carries ~105 MB more filter blocks (copied + CRC32C'd as they are); measured on the build "
                "container's CPU, not on the GPU box"}, indent=1))


if __name__ == "__main__":
    main()
