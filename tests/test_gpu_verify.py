"""The output check on the GPU (ybgpu_job_verify_output, ybgpu_sst_verify_device, the *_checked pipelines): every job
shape the parity and route suites generate verifies clean with the oracle's counts, and damaged tables are caught on the
device with the kind, block and entry the CPU judgement (tests/test_verify_cpu.py) reports for the same bytes."""
import importlib
import os
import subprocess

import pytest

import oracle_py as o
import verify_util as vu
import workloads as w
from test_gpu_parity import _phrase_runs, _stored_types, gpu_compact, okw, runs_to_ssts
from test_gpu_routes import docdb_wide_runs, has, lacks

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    m = importlib.import_module("yugabyte-db_b200")
    assert m.device_count() >= 1, "GPU tests need a CUDA device"
    return m


def verified(pkg, ssts, block_size=4096, ht_filters=None, **kw):
    """One job against the oracle, then checked on the device: OK, flagged, the oracle's counts, and the files it
    fetches afterwards still the oracle's."""
    topt = o.TableOptions(block_size=block_size, key_encoding=kw.get("output_key_encoding", 1),
                          filter_policy=kw.get("filter_policy", 0), filter_block_size=kw.get("filter_block_size", 65536),
                          compression=kw.get("output_compression", 0))
    exp = o.compact(ssts, o.CompactionParams(**okw(kw)), topt, ht_filters=ht_filters)
    job = gpu_compact(pkg, ssts, ht_filters=ht_filters, block_size=block_size, **kw)
    assert lacks(job.stats(), pkg.PATH_OUTPUT_VERIFIED)
    chk = job.verify_output()
    assert chk.failure_kind == 0 and has(job.stats(), pkg.PATH_OUTPUT_VERIFIED)
    ref = exp.sst()
    data, meta = job.fetch_output()
    if ref is None:
        assert (chk.blocks_checked, chk.entries_parsed, chk.blocks_compressed) == (0, 0, 0) and data.size == 0
        return job, chk
    assert data.tobytes() == ref.data and meta.tobytes() == ref.meta
    types, _, _ = _stored_types(ref.data, ref.meta, pkg)
    assert chk.blocks_checked == len(types)
    assert chk.entries_parsed == exp.stats.num_output_records == job.stats().num_output_records
    assert chk.blocks_compressed == sum(1 for t in types if t)
    assert chk.bytes_read >= len(ref.data) and chk.gpu_seconds > 0
    again = job.verify_output()                                   # any number of times, also after the fetch
    assert (again.blocks_checked, again.entries_parsed, again.failure_kind) == (chk.blocks_checked, chk.entries_parsed, 0)
    return job, chk


def test_illegal_state_before_run(pkg):
    job = pkg.GpuCompactionJob()
    with pytest.raises(pkg.YbGpuError) as e:
        job.verify_output()
    assert e.value.status_name == "IllegalState"


def test_config1_and_generated_mvcc_heavy(pkg):
    cfg = o.GenConfig(seed=5, num_rows=3000, cols=3, versions=6, num_files=4, value_len=200, tombstone_per_1024=100)
    ssts = o.Sst.generate_all(cfg, o.TableOptions(block_size=32768))
    for cut in (0, 2500, 10**7):
        job, chk = verified(pkg, ssts, block_size=32768, cutoff_ht=o.ht_from_micros(cfg.base_micros + cut))
        assert has(job.stats(), pkg.PATH_ENCODER_V5)
    verified(pkg, ssts, block_size=32768, bottommost=False, cutoff_ht=o.HT_MIN, other_min_ht=o.HT_MIN)


@pytest.mark.parametrize("seed", range(4))
def test_randomized_docdb_retention_grid(pkg, seed):
    """TTL merges and expirations: rewritten value prefixes and values turned into tombstones are compared too."""
    runs = w.random_docdb_runs(seed, n_runs=1 + seed % 5, n_rows=150 + 40 * seed)
    ssts = runs_to_ssts(runs, 512 if seed % 2 else 2048)
    for kw in w.param_grid():
        verified(pkg, ssts, block_size=1024, output_key_encoding=1 + seed % 2, **kw)


def test_wide_keys_v4_and_fused_encoders(pkg):
    for width in (281, 1016):
        dssts = runs_to_ssts(docdb_wide_runs(1000 + width, width), 1024)
        for enc in (1, 2):
            job, _ = verified(pkg, dssts, block_size=4096, output_key_encoding=enc, **w.param_grid()[2])
            assert has(job.stats(), pkg.PATH_ENCODER_V4) and lacks(job.stats(), pkg.PATH_ENCODER_V5)
        big = runs_to_ssts(docdb_wide_runs(4000 + width, width, n_rows=600), 4096)
        job, _ = verified(pkg, big, block_size=65536, **w.param_grid()[0])
        assert has(job.stats(), pkg.PATH_ENCODER_FUSED)
        verified(pkg, dssts, block_size=4096, output_compression=1, **w.param_grid()[2])


def test_rows_larger_than_a_merge_tile_and_colocated(pkg):
    runs = w.giant_row_runs(1, cols=120, versions=45, collection=1500, colocated=True)
    verified(pkg, runs_to_ssts(runs, 4096), **w.param_grid()[2])
    for seed in range(3):
        ssts = runs_to_ssts(w.random_cotable_runs(seed, colocated=bool(seed % 2)), 1024)
        for kw in (w.param_grid()[0], w.param_grid()[2]):
            verified(pkg, ssts, block_size=1024, **kw)


@pytest.mark.parametrize("compression", [1, 4])
def test_compressed_outputs_mixed_with_raw_blocks(pkg, compression):
    runs = _phrase_runs(901, 1, 3000, vmax=400, random_every=300)   # one run: the stretches of random values stay together
    ssts = [o.Sst.build(r, o.TableOptions(block_size=4096, compression=1)) for r in runs if r]
    for enc in (1, 2):
        job = gpu_compact(pkg, ssts, block_size=4096, output_key_encoding=enc, output_compression=compression, **w.param_grid()[0])
        chk = job.verify_output()
        data, meta = job.fetch_output()
        types, _, _ = _stored_types(data.tobytes(), meta.tobytes(), pkg)
        assert 0 < chk.blocks_compressed == sum(1 for t in types if t) < chk.blocks_checked == len(types)
        assert chk.entries_parsed == job.stats().num_output_records and has(job.stats(), pkg.PATH_OUTPUT_VERIFIED)
        assert pkg.sst_verify_device(meta, data).entries_parsed == chk.entries_parsed
    if compression == 1:
        verified(pkg, ssts, block_size=4096, output_compression=1, filter_policy=1, filter_block_size=4096, **w.param_grid()[2])


def test_kv_stream_inputs_empty_output_and_single_entry(pkg):
    runs = w.random_docdb_runs(11, n_runs=3, n_rows=200)
    exp = o.compact(runs_to_ssts(runs), o.CompactionParams(retention=False), o.TableOptions(block_size=1024))
    job = pkg.GpuCompactionJob(retention=False, block_size=1024)
    for r in runs:
        job.add_input_kv(r)
    job.run()
    chk = job.verify_output()
    assert has(job.stats(), pkg.PATH_KV_INPUT, pkg.PATH_OUTPUT_VERIFIED) and chk.entries_parsed == exp.stats.num_output_records
    assert job.fetch_output()[0].tobytes() == exp.sst().data
    # everything deleted at the bottommost level: no table, zero counts
    dead = [(o.ikey(b"k%03d" % i, 10 + i, 0), b"") for i in range(50)]
    _, chk = verified(pkg, [o.Sst.build(dead, o.TableOptions(block_size=1024))], retention=False, bottommost=True)
    assert chk.blocks_checked == 0
    _, chk = verified(pkg, [o.Sst.build([(o.ikey(b"only", 7), b"v")])], retention=False)
    assert (chk.blocks_checked, chk.entries_parsed) == (1, 1)


def _device(pkg, t):
    try:
        chk = pkg.sst_verify_device(t.meta, bytes(t.data))
        return (0, 0, 0), chk.entries_parsed
    except pkg.OutputCheckError as e:
        assert e.status_name == "Corruption"
        return (e.check.failure_kind, e.check.failure_block, e.check.failure_entry), None


def test_damaged_tables_are_caught_on_the_device(pkg):
    """The CPU sweep's tables through ybgpu_sst_verify_device: the same verdict, and a good table still passes afterwards."""
    kvs = vu.rand_kvs(41, 1200)
    for restart in (1, 16):
        t = vu.build_table(pkg, kvs, 1, restart, 2048)
        assert _device(pkg, t) == ((0, 0, 0), len(kvs))
        caught = set()
        for b in (0, len(t.offs) // 2, len(t.offs) - 1):
            for seed in range(3):
                for name, m in vu.byte_mutations(t, b, 1000 * b + seed).items():
                    want, _ = vu.cpu_check(m)
                    got, _ = _device(pkg, m)
                    assert got == want, (restart, name, b, seed)
                    caught.add(vu.KINDS[got[0]])
            m = t.copy()
            m.data[t.offs[b] + t.sizes[b] // 2] ^= 0x10                # not re-sealed
            assert _device(pkg, m)[0] == (1, b, 0)
        assert {"entry_parse", "key_order", "ok"} <= caught
        assert _device(pkg, t) == ((0, 0, 0), len(kvs))
    for enc, compression in ((1, 0), (2, 0), (1, 1), (2, 4)):
        good = vu.build_table(pkg, kvs, enc, 16, 2048, compression)
        assert _device(pkg, good) == ((0, 0, 0), len(kvs))
        bf = vu.block_first(good)
        b = len(bf) // 2
        for name, bad_kvs in vu.kv_mutations(kvs, bf, b).items():
            m = vu.build_table(pkg, bad_kvs, enc, 16, 2048, compression)
            want, _ = vu.cpu_check(m)
            assert (want[0] == 0) == (name in ("dropped", "truncated"))
            assert _device(pkg, m)[0] == want, (enc, compression, name)
        if compression:
            m = good.copy()
            m.data[good.offs[b] + good.sizes[b] // 2] ^= 0x10
            assert _device(pkg, m)[0] == (1, b, 0)
            m.reseal(b)
            want, _ = vu.cpu_check(m)
            assert _device(pkg, m)[0] == want
        assert _device(pkg, good) == ((0, 0, 0), len(kvs))


def test_checked_pipelines_give_the_same_files(pkg):
    runs = w.random_docdb_runs(21, n_runs=4, n_rows=2500)
    tables = runs_to_ssts(runs, 4096)                     # the views below point into these
    ssts = [(s.meta_view(), s.data_view()) for s in tables]
    kw = dict(block_size=4096, filter_policy=1, filter_block_size=4096, output_compression=1, **w.param_grid()[2])
    plain = pkg.compact_files(ssts, max_subcompactions=8, max_in_flight=3, **kw)
    checked = pkg.compact_files(ssts, max_subcompactions=8, max_in_flight=3, verify_outputs=True, **kw)
    unchecked = pkg.compact_files(ssts, max_subcompactions=8, max_in_flight=3, verify_outputs=False, **kw)
    assert len(plain.outputs) == len(checked.outputs) == 8
    assert [(bytes(d), bytes(m)) for d, m in checked.files()] == [(bytes(d), bytes(m)) for d, m in plain.files()]
    for oc, op, ou in zip(checked.outputs, plain.outputs, unchecked.outputs):
        assert oc.stats.path_flags & pkg.PATH_OUTPUT_VERIFIED or not oc.stats.num_output_records
        assert not op.stats.path_flags & pkg.PATH_OUTPUT_VERIFIED and not ou.stats.path_flags & pkg.PATH_OUTPUT_VERIFIED
    d0, m0, r0, t0 = pkg.compact_files_one_table(ssts, max_subcompactions=8, max_in_flight=3, **kw)
    d1, m1, r1, t1 = pkg.compact_files_one_table(ssts, max_subcompactions=8, max_in_flight=3, verify_outputs=True, **kw)
    assert bytes(d0) == bytes(d1) and bytes(m0) == bytes(m1) and r1.num_ranges == 8
    assert t1.path_flags & pkg.PATH_OUTPUT_VERIFIED and not t0.path_flags & pkg.PATH_OUTPUT_VERIFIED
    assert pkg.sst_verify_device(m1, d1).entries_parsed == t1.num_output_records


def test_adapter_paranoid_file_checks(pkg, tmp_path):
    """Params::paranoid_file_checks: Run() checks the table on the device, single job and one job per key range."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe, lib_dir = str(tmp_path / "adapter_verify_test"), os.path.join(root, "yugabyte-db_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(root, "tests", "adapter_verify_test.cc"),
                           "-L" + lib_dir, "-lybgpu", "-Wl,-rpath," + lib_dir, "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64"])
    runs = _phrase_runs(905, 3, 1200)
    args = []
    for i, r in enumerate(runs):
        s = o.Sst.build(r, o.TableOptions(block_size=4096, compression=1))
        for ext, blob in ((".sst", s.meta), (".sst.sblock.0", s.data)):
            path = tmp_path / ("%d%s" % (i, ext))
            path.write_bytes(blob)
            args.append(str(path))
    parsed = set()
    for nsub in (1, 4):
        out = subprocess.check_output([exe, str(nsub)] + args, text=True).split()
        assert out[0] == "OK" and int(out[1]) > 0 and int(out[2]) == (1 if nsub == 1 else 4), out
        parsed.add(int(out[1]))
    assert len(parsed) == 1                      # the same survivors either way
