"""What colocated tables cost the merge. Usage: python profiles/colocated_measure.py [--tables N]

About 20 000 colocated tables ('0' + u32 colocation id), 1-60 rows each with 1-2 versions of 2 columns, a tenth of
them with 1-5 table-tombstone versions, in 4 input files written by the product's host table builder
(ybgpu_table_builder_*): about 2 M entries. The same rows with the ids stripped (every key an id-less DocKey naming its
table in a range component; no table tombstones) are the arm that the merge kernel handles without any table state.
Each arm is compacted three times, alternated: merge phase (phase_seconds[3]), all device phases (gpu_seconds) and the
host wall clock of the whole job (inputs added, run, outputs fetched). Prints the card and its power limit first."""
import importlib
import os
import random
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]
pkg = importlib.import_module("yugabyte-db_b200")
import dockv_util as dk        # noqa: E402
import oracle_py as o          # noqa: E402

if pkg.device_count() < 1:
    raise SystemExit("colocated_measure.py needs a CUDA device")

print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
n_tables = int(sys.argv[sys.argv.index("--tables") + 1]) if "--tables" in sys.argv else 20000
BASE_US = o.YB_EPOCH_US + 100_000_000
N_FILES = 4


def build_inputs(stripped):
    rng = random.Random(17)
    runs = [[] for _ in range(N_FILES)]
    seq = [(1 << 50) + (r << 32) for r in range(N_FILES)]
    cols = [dk.kcol(1), dk.kcol(2)]
    for t in range(n_tables):
        kw = {} if stripped else dict(colocation=16384 + t)
        if not stripped and rng.random() < 0.1:
            for m in rng.sample(range(200), rng.randrange(1, 6)):
                r = rng.randrange(N_FILES)
                seq[r] += 1
                runs[r].append((dk.table_tombstone_key(micros=BASE_US + m, **kw), seq[r], dk.TOMBSTONE))
        for row in range(rng.randrange(1, 61)):
            d = dk.doc_key(["t%05d" % t, row] if stripped else [row], **kw)
            for c in cols:
                for _ in range(rng.randrange(1, 3)):
                    uk = dk.sub_doc_key(d, [c], micros=BASE_US + rng.randrange(200), logical=rng.randrange(4))
                    r = rng.randrange(N_FILES)
                    seq[r] += 1
                    runs[r].append((uk, seq[r], dk.vstr("value-%08d" % rng.randrange(10**8))))
    files = []
    for run in runs:
        run.sort(key=lambda e: (e[0], -e[1]))
        b = pkg.HostTableBuilder(block_size=32768)
        last = None
        for uk, s, v in run:
            if uk == last:                   # one version per user key (a random HT can repeat)
                continue
            last = uk
            b.add(o.ikey(uk, s), v)
        data, meta = b.finish()
        files.append((np.frombuffer(meta, np.uint8), np.frombuffer(data, np.uint8)))
    return files


def run_job(files):
    t0 = time.perf_counter()
    job = pkg.GpuCompactionJob(cutoff_ht=o.ht_from_micros(BASE_US + 100), bottommost=False)
    for meta, data in files:
        job.add_input_sst(meta, data)
    job.run()
    job.fetch_output()
    wall = time.perf_counter() - t0
    st = job.stats()
    job.close()
    return st, wall


arms = {"colocated": build_inputs(False), "ids stripped": build_inputs(True)}
for name, files in arms.items():
    print("%-13s %d input bytes" % (name, sum(len(d) for _, d in files)))
for name, files in arms.items():                      # warm-up
    try:
        run_job(files)
    except pkg.YbGpuError as e:
        print("%-13s fails: %s" % (name, e))
for rep in range(3):
    for name, files in arms.items():
        try:
            st, wall = run_job(files)
        except pkg.YbGpuError as e:
            print("%-13s fails: %s" % (name, e))
            continue
        print("%-13s %d entries -> %d: merge %.3f ms, device %.3f ms, whole job %.1f ms" % (
            name, st.num_input_records, st.num_output_records, st.phase_seconds[3] * 1e3, st.gpu_seconds * 1e3, wall * 1e3))
