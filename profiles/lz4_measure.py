"""What LZ4 costs on the GPU next to Snappy, in one run on one card. Usage: python profiles/lz4_measure.py

Output side: the generator's shapes (256-byte random values: nothing compresses and every position is visited; 16-byte
values: keys dominate and blocks compress; tombstone-heavy tables), each compacted with output compression none, Snappy
and LZ4, alternated, twice: device time of the block compressor and of the gather (stats slots 6 / 7) and the stored /
raw ratio. Input side: the same tables compacted once with output compression 1 and once with 4 give Snappy and LZ4
inputs; compacting those (raw output), and the uncompressed table as a baseline, times phase 0, the block scan that
holds the uncompress stage. Prints the card and its power limit first."""
import importlib
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]
pkg = importlib.import_module("yugabyte-db_b200")
if pkg.device_count() < 1:
    raise SystemExit("lz4_measure.py needs a CUDA device")

print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())


def compact(inputs, comp):
    job = pkg.GpuCompactionJob(output_compression=comp, retain_delete_markers=True)
    for m, d in inputs:
        job.add_input_sst(m, d)
    job.run()
    st = job.stats()
    data, meta = job.fetch_output()
    return st, data.copy(), meta.copy()


NAMES = {0: "none  ", 1: "snappy", 4: "lz4   "}
for value_len, rows, tomb in ((256, 4000000, 0), (16, 8000000, 0), (64, 6000000, 700)):
    cfg = pkg.GenConfig(seed=7, num_rows=rows, cols=1, versions=1, num_files=4, value_len=value_len, tombstone_per_1024=tomb, tombstone_newest=1)
    gens = pkg.generate_ssts(cfg)
    files = [(g.meta_view(), g.data_view()) for g in gens]
    print("== value_len %d, tombstones %d/1024, %d rows" % (value_len, tomb, rows))
    raw_size, outs = None, {}
    for rep in range(2):
        for comp in (0, 1, 4):
            st, data, meta = compact(files, comp)
            if comp == 0:
                raw_size = data.size
                print("  %s output phase %.3f ms, %d bytes" % (NAMES[comp], st.phase_seconds[4] * 1e3, data.size))
                outs[comp] = (meta, data)
            else:
                cms, gms = st.phase_seconds[6] * 1e3, st.phase_seconds[7] * 1e3
                print("  %s encoder %.3f ms (%.1f GB/s of block bytes), gather %.3f ms, output phase %.3f ms, stored/raw %.3f"
                      % (NAMES[comp], cms, raw_size / max(cms, 1e-6) / 1e6, gms, st.phase_seconds[4] * 1e3, data.size / raw_size))
                outs[comp] = (meta, data)
    # inputs stored with each codec: the block-scan phase (checksums, probe, uncompress into one image, probe again)
    for rep in range(2):
        for comp in (0, 1, 4):
            st, _, _ = compact([outs[comp]], 0)
            print("  %s inputs: block scan + uncompress (phase 0) %.3f ms, flags %#x" % (NAMES[comp], st.phase_seconds[0] * 1e3, st.path_flags))
    del gens, files, outs
