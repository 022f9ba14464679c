"""Colocated ('0' + u32 colocation id) and cotable ('y' + uuid) tablets with any number of tables per merge tile and any
number of table-tombstone versions per table. A table tombstone `id ! # HT` sets slot 0 of DocDBCompactionFeed's overwrite
stack for every row of its table (docdb_compaction_context.cc:999-1024). The merge kernel takes that state from the
tile's own records, and looks it up in the runs only for the table the tile starts in. Every case is checked against
the oracle: KV stream, counters, digest, boundaries and both output files."""
import importlib
import random
import struct

import pytest

import dockv_util as dk
import oracle_py as o
import workloads as w
from test_gpu_parity import check, okw, runs_to_ssts

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    m = importlib.import_module("yugabyte-db_b200")
    assert m.device_count() >= 1, "GPU tests need a CUDA device"
    return m


def table_id(t, colocated):
    """Keyword arguments of dk.doc_key / dk.table_tombstone_key for table t: colocation id, or a cotable uuid whose
    last four bytes (the database oid of the per-database HybridTime filters) take 8 values."""
    if colocated:
        return dict(colocation=1000 + 7 * t)
    return dict(cotable=struct.pack(">I", 0x10000 + t) + bytes([(t * 37 + j) % 251 + 1 for j in range(8)]) + struct.pack("<I", 100 + t % 8))


class Runs:
    """Sorted runs under construction: each entry goes to a random run (or to `run`) with a fresh sequence number."""

    def __init__(self, rng, n_runs):
        self.rng, self.runs = rng, [[] for _ in range(n_runs)]
        self.seq = [(1 << 50) + (r << 30) for r in range(n_runs)]
        self.used = set()

    def put(self, user_key, value, run=None):
        if user_key in self.used:
            return
        self.used.add(user_key)
        r = self.rng.randrange(len(self.runs)) if run is None else run
        self.seq[r] += 1
        self.runs[r].append((o.ikey(user_key, self.seq[r]), value))

    def sorted(self):
        return [w.sort_run(r) for r in self.runs]


def put_rows(R, rng, kw, n_rows, n_ht=12, tag="r"):
    for row in range(n_rows):
        d = dk.doc_key(["%s%03d" % (tag, row)], **kw) if rng.random() < 0.5 else \
            dk.doc_key([row], hash_code=rng.randrange(65536), hashed=["h%d" % row], **kw)
        for c in range(rng.randrange(1, 3)):
            for _ in range(rng.randrange(1, 3)):
                ht = (w.BASE_US + rng.randrange(n_ht) * 10, rng.randrange(2), 0)
                R.put(dk.sub_doc_key(d, [dk.kcol(c + 1)], ht=ht), dk.TOMBSTONE if rng.random() < 0.15 else dk.vstr("v%d" % rng.randrange(1000)))


def put_tombstones(R, rng, kw, n, run=None):
    """n versions of the table's tombstone at distinct hybrid times, on both sides of param_grid()'s cutoffs."""
    for m in rng.sample(range(max(2 * n, 120)), n):
        R.put(dk.table_tombstone_key(micros=w.BASE_US + m, **kw), dk.TOMBSTONE, run=run)


def many_tables_runs(seed, n_tables=2000, colocated=True, n_runs=4):
    """n_tables small tables (1-4 rows each, 0-3 tombstone versions): a merge tile spans hundreds of tables."""
    rng = random.Random(seed)
    R = Runs(rng, n_runs)
    for t in range(n_tables):
        kw = table_id(t, colocated)
        put_tombstones(R, rng, kw, rng.choice([0, 0, 1, 2, 3]))
        put_rows(R, rng, kw, rng.randrange(1, 5))
    return R.sorted()


def many_versions_runs(seed, n_tables=40, colocated=True, n_runs=4, versions=(20, 60), rows=(20, 120), tomb_run=None):
    """Tables with 20-60 tombstone versions spread over the runs (or all in run `tomb_run`), and enough rows that merge
    tiles start inside tables."""
    rng = random.Random(seed)
    R = Runs(rng, n_runs)
    for t in range(n_tables):
        kw = table_id(t, colocated)
        put_tombstones(R, rng, kw, rng.randrange(*versions), run=tomb_run)
        put_rows(R, rng, kw, rng.randrange(*rows), n_ht=20)
    return R.sorted()


def mixed_runs(seed, n_runs=3):
    """Rows of tables with and without tombstones, cotable and colocated ids, interleaved with id-less rows."""
    rng = random.Random(seed)
    R = Runs(rng, n_runs)
    for t in range(300):
        kw = table_id(t, t % 2 == 0)
        if t % 3 == 0:
            put_tombstones(R, rng, kw, rng.randrange(1, 25))
        put_rows(R, rng, kw, rng.randrange(0, 6))
    for row in range(1500):
        d = dk.doc_key(["plain%05d" % row]) if row % 2 else dk.doc_key([row], hash_code=rng.randrange(65536), hashed=["h%d" % row])
        R.put(dk.sub_doc_key(d, [dk.kcol(1)], ht=(w.BASE_US + rng.randrange(12) * 10, 0, 0)), dk.vstr("p%d" % row))
    return R.sorted()


@pytest.mark.parametrize("colocated", [True, False])
@pytest.mark.parametrize("n_runs", [1, 3, 8])
def test_many_small_tables(pkg, colocated, n_runs):
    runs = many_tables_runs(n_runs + 10 * colocated, colocated=colocated, n_runs=n_runs)
    ssts = runs_to_ssts(runs, 1024)
    for kw in w.param_grid():
        check(pkg, ssts, block_size=1024, **kw)
    if not colocated:                  # 'y' keys under the master's cotables history cutoff
        check(pkg, ssts, block_size=1024, bottommost=True, cutoff_ht=o.ht_from_micros(w.BASE_US + 35),
              cotables_cutoff_ht=o.ht_from_micros(w.BASE_US + 85))


@pytest.mark.parametrize("seed", range(4))
def test_many_tombstone_versions(pkg, seed):
    """20-60 table-tombstone versions per table. Tiles start inside the tables' rows, so the tile's first table takes
    its tombstones from the runs."""
    runs = many_versions_runs(seed, colocated=seed % 2 == 0, n_runs=1 + 2 * seed)
    ssts = runs_to_ssts(runs, 256)
    for kw in w.param_grid():
        check(pkg, ssts, block_size=256, **kw)


@pytest.mark.parametrize("colocated", [True, False])
def test_tiles_start_inside_the_tombstones(pkg, colocated):
    """Tombstone groups longer than a run's sample stride (all versions in one of 8 runs) and one of 3 000 versions,
    longer than a merge tile: tiles start inside tombstone groups, and only those groups are that long."""
    runs = many_versions_runs(7 + colocated, n_tables=10, colocated=colocated, n_runs=8, versions=(150, 400), rows=(5, 40), tomb_run=3)
    R = Runs(random.Random(3), 8)
    kw = table_id(5000, colocated)
    for m in range(3000):
        R.put(dk.table_tombstone_key(micros=w.BASE_US + m, **kw), dk.TOMBSTONE)
    put_rows(R, random.Random(4), kw, 60, n_ht=20)
    runs = [a + b for a, b in zip(runs, R.runs)]
    ssts = runs_to_ssts([w.sort_run(r) for r in runs], 512)
    grid = w.param_grid()
    for kw in [grid[i] for i in (0, 1, 2, 3, 4, 6, 8, 9, 10)]:
        job, _ = check(pkg, ssts, block_size=512, **kw)
        assert job.stats().tiles_inside_rows > 0


@pytest.mark.parametrize("seed", range(3))
def test_mixed_keys(pkg, seed):
    runs = mixed_runs(seed, n_runs=2 + seed)
    ssts = runs_to_ssts(runs, 1024)
    for kw in w.param_grid()[::2]:
        check(pkg, ssts, block_size=1024, **kw)


def _range_outputs(res):
    got = []
    for out in res.outputs:
        if out.data_len:
            got += o.Sst.from_bytes(res.meta_arena[out.meta_offset:out.meta_offset + out.meta_len].tobytes(),
                                    res.data_arena[out.data_offset:out.data_offset + out.data_len].tobytes()).read_all()
    return got


@pytest.mark.parametrize("colocated", [True, False])
def test_key_ranges_inside_tables(pkg, colocated):
    """compact_files and compact_files_one_table over many small tables: ranges start inside tables, whose tombstones
    are loaded out of range and seed the rows. The range outputs concatenate to the single-job stream."""
    runs = many_tables_runs(40 + colocated, n_tables=800, colocated=colocated, n_runs=3)
    runs = [a + b for a, b in zip(runs, many_versions_runs(50 + colocated, n_tables=6, colocated=colocated, n_runs=3))]
    ssts = runs_to_ssts([w.sort_run(r) for r in runs], 512)
    files = [(s.meta_view(), s.data_view()) for s in ssts]
    inside = 0
    for kw in [w.param_grid()[i] for i in (0, 2, 4, 7, 9)]:
        exp = o.compact(ssts, o.CompactionParams(**okw(kw)), o.TableOptions(block_size=1024))
        res = pkg.compact_files(files, max_subcompactions=9, max_in_flight=2, block_size=1024, **kw)
        assert len(res.outputs) >= 7
        for out in res.outputs:
            if out.lower and out.lower[:1] in (b"y", b"0") and len(out.lower) > (17 if out.lower[:1] == b"y" else 5) + 1:
                inside += 1
        assert _range_outputs(res) == exp.kv_list()
        assert res.total.num_input_records == exp.stats.num_input_records
        assert res.total.num_output_records == exp.stats.num_output_records
        assert res.total.num_record_drop_feed == exp.stats.num_dropped_feed
        data, meta, one, total = pkg.compact_files_one_table(files, max_subcompactions=7, max_in_flight=2, block_size=1024, **kw)
        ekv = exp.kv_list()
        assert o.Sst.from_bytes(meta.tobytes(), data.tobytes()).read_all() == ekv
        assert (one.smallest, one.largest) == ((ekv[0][0], ekv[-1][0]) if ekv else (b"", b""))
        assert total.num_input_records == exp.stats.num_input_records and total.num_output_records == exp.stats.num_output_records
    assert inside >= 7, "the ranges must start inside tables"


def test_key_ranges_with_cotable_filters(pkg):
    """Per-database cotable HybridTime filters: filtered tombstones do not seed the rows, out-of-range ones do."""
    runs = many_versions_runs(60, n_tables=16, colocated=False, n_runs=3, versions=(20, 40), rows=(10, 60))
    ssts = runs_to_ssts(runs, 512)
    f_lo, f_mid = o.ht_from_micros(w.BASE_US + 15), o.ht_from_micros(w.BASE_US + 30, 1)
    cot = [([100, 103, 106], [f_lo, f_mid, f_lo]), ([101, 103], [f_mid, f_lo]), ([], [])]
    glob = [o.HT_INVALID, o.ht_from_micros(w.BASE_US + 45), o.HT_INVALID]
    files = [(s.meta_view(), s.data_view()) for s in ssts]
    for kw in [w.param_grid()[i] for i in (0, 2, 3, 5)]:
        exp = o.compact(ssts, o.CompactionParams(**kw), o.TableOptions(block_size=1024), ht_filters=glob, cotable_filters=cot)
        job = pkg.GpuCompactionJob(block_size=1024, **kw)
        for i, s in enumerate(ssts):
            job.add_input_sst(s.meta_view(), s.data_view(), ht_filter=glob[i])
            job.set_cotable_filters(*cot[i])
        job.run()
        assert job.kv_list() == exp.kv_list()
        st = job.stats()
        assert (st.num_input_records, st.num_output_records) == (exp.stats.num_input_records, exp.stats.num_output_records)
        assert st.num_record_drop_feed == exp.stats.num_dropped_feed
        data, meta = job.fetch_output()
        ref = exp.sst()
        assert (data.tobytes(), meta.tobytes()) == ((ref.data, ref.meta) if ref is not None else (b"", b""))
        res = pkg.compact_files(files, max_subcompactions=8, max_in_flight=2, ht_filters=glob, cotable_filters=cot, block_size=1024, **kw)
        assert len(res.outputs) >= 6
        assert _range_outputs(res) == exp.kv_list()
        assert res.total.num_output_records == exp.stats.num_output_records


def test_flush_of_a_colocated_memtable(pkg):
    """add_input_kv: the flush path's input, one colocated memtable with many tables."""
    mem = many_tables_runs(70, n_tables=1500, colocated=True, n_runs=1)[0]
    ssts = runs_to_ssts([mem], 1024)
    for kw in (w.param_grid()[1], w.param_grid()[3], w.param_grid()[10]):
        exp = o.compact(ssts, o.CompactionParams(**kw), o.TableOptions(block_size=2048))
        job = pkg.GpuCompactionJob(block_size=2048, **kw)
        job.add_input_kv(mem)
        job.run()
        st = job.stats()
        assert st.path_flags & pkg.PATH_KV_INPUT
        assert job.kv_list() == exp.kv_list()
        assert (st.num_input_records, st.num_output_records) == (exp.stats.num_input_records, exp.stats.num_output_records)
        assert st.num_record_drop_feed == exp.stats.num_dropped_feed
        assert job.digest() == exp.stats.kv_hash
        data, meta = job.fetch_output()
        ref = exp.sst()
        assert (data.tobytes(), meta.tobytes()) == ((ref.data, ref.meta) if ref is not None else (b"", b""))
