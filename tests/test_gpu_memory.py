"""Device memory accounting and budgets on the GPU: ybgpu_job_stats::device_bytes_peak against the stream-ordered pool's
own high-water mark on every route shape, budgets of exactly the peak and one byte less, the refusal before upload, and
pipelined compactions planned and re-cut to fit a budget, all against the oracle."""
import ctypes as C
import importlib

import pytest

import lz4_util as z
import oracle_py as o
import workloads as w
from test_gpu_parity import _phrase_runs

pytestmark = pytest.mark.gpu



@pytest.fixture(scope="module")
def pkg():
    m = importlib.import_module("yugabyte-db_b200")
    assert m.device_count() >= 1, "GPU tests need a CUDA device"
    return m


class Pool:
    """cudaMemPoolAttrUsedMemCurrent / UsedMemHigh of device 0's default pool (the pool the engine allocates from)."""
    USED_CURRENT, USED_HIGH = 7, 8

    def __init__(self, pkg):
        pkg.lib()                                    # libcudart is loaded with the engine
        self.rt = C.CDLL("libcudart.so.12")
        self.pool = C.c_void_p()
        assert self.rt.cudaDeviceGetDefaultMemPool(C.byref(self.pool), 0) == 0

    def _get(self, attr):
        v = C.c_uint64()
        assert self.rt.cudaMemPoolGetAttribute(self.pool, attr, C.byref(v)) == 0
        return v.value

    def used(self):
        assert self.rt.cudaDeviceSynchronize() == 0
        return self._get(self.USED_CURRENT)

    def reset_high(self):
        assert self.rt.cudaDeviceSynchronize() == 0
        zero = C.c_uint64(0)
        assert self.rt.cudaMemPoolSetAttribute(self.pool, self.USED_HIGH, C.byref(zero)) == 0
        return self._get(self.USED_CURRENT)

    def high(self):
        assert self.rt.cudaDeviceSynchronize() == 0
        return self._get(self.USED_HIGH)


@pytest.fixture(scope="module")
def pool(pkg):
    return Pool(pkg)


def _cfg_runs(seed, num_rows=3000, value_len=120):
    cfg = o.GenConfig(seed=seed, num_rows=num_rows, cols=2, versions=3, num_files=3, value_len=value_len, tombstone_per_1024=40)
    return cfg, [s.read_all() for s in o.Sst.generate_all(cfg, o.TableOptions(block_size=4096))]


def _shapes(pkg):
    """(name, tables or None, kv runs or None, job kwargs, verify_output) for every route the engine picks by input shape."""
    cfg, runs = _cfg_runs(5)
    kw = dict(cutoff_ht=o.ht_from_micros(cfg.base_micros + 1500), block_size=4096)
    raw = [o.Sst.build(r, o.TableOptions(block_size=4096)) for r in runs]
    tsp = [o.Sst.build(r, o.TableOptions(block_size=2048, key_encoding=2)) for r in runs]
    phrases = _phrase_runs(31, 3, 600)
    snappy = [o.Sst.build(r, o.TableOptions(block_size=4096, compression=1)) for r in phrases]
    lz4 = [z.host_lz4_table(pkg, r, block_size=4096) for r in phrases]
    cot = [r for r in w.random_cotable_runs(17, n_runs=3, n_tables=6, rows_per_table=40) if r]
    cot_t = [o.Sst.build(r, o.TableOptions(block_size=2048)) for r in cot]
    return [
        ("fused", raw, None, kw, False),
        ("general_decode", tsp, None, kw, False),
        ("snappy_in", snappy, None, kw, False),
        ("lz4_in", lz4, None, kw, False),
        ("snappy_out", raw, None, dict(kw, output_compression=1), False),
        ("lz4_out", snappy, None, dict(kw, output_compression=4), False),
        ("filters", raw, None, dict(kw, filter_policy=1, filter_block_size=4096), False),
        ("verify_output", raw, None, dict(kw, output_compression=1), True),
        ("kv_inputs", None, runs, dict(kw, retention=False), False),
        ("colocated", cot_t, None, dict(block_size=2048, cutoff_ht=o.ht_from_micros(1790000000 * 1000000 + 6)), False),
    ]


def _run(pkg, tables, kvs, kw, verify, budget=0, job=None):
    job = job or pkg.GpuCompactionJob(device_memory_budget=budget, **kw)
    if tables is not None:
        for s in tables:
            job.add_input_sst(s.meta_view(), s.data_view())
    else:
        for r in kvs:
            job.add_input_kv(r)
    job.run()
    if verify:
        job.verify_output()
    return job


def _result(job):
    data, meta = job.fetch_output()
    return job.kv_list(), data.tobytes(), meta.tobytes()


def test_peak_matches_the_pool_and_budgets_hold_on_every_route(pkg, pool):
    """device_bytes_peak == the pool's UsedMemHigh delta (the pool counts requested bytes, so an allocation that bypassed
    the job's accounting would show as a difference); a budget of exactly the peak gives
    the same KV stream and files, one byte less fails with the budget message, and afterwards a job with the peak as its
    budget runs again and the pool's used bytes come back to where they started."""
    for name, tables, kvs, kw, verify in _shapes(pkg):
        base = pool.reset_high()
        job = _run(pkg, tables, kvs, kw, verify)
        want = _result(job)                          # the KV stream fetch allocates too: the peak is taken after it
        peak = job.stats().device_bytes_peak
        delta = pool.high() - base
        assert 0 < peak == delta, (name, peak, delta)
        if name in ("snappy_in", "lz4_in"):
            assert job.stats().path_flags & (pkg.PATH_SNAPPY | pkg.PATH_LZ4), name
        job.close()
        assert pool.used() == base, name

        same = _run(pkg, tables, kvs, kw, verify, budget=peak)
        assert _result(same) == want, name
        assert same.stats().device_bytes_peak == peak, name
        same.close()

        short = pkg.GpuCompactionJob(device_memory_budget=peak - 1, **kw)
        with pytest.raises(pkg.YbGpuError) as ei:
            _result(_run(pkg, tables, kvs, kw, verify, job=short))
        short.close()
        assert "device memory budget exceeded: need" in str(ei.value) and "budget %d" % (peak - 1) in str(ei.value), name
        assert ei.value.status_name in ("RuntimeError", "NotSupported"), name
        assert pool.used() == base, name
        again = _run(pkg, tables, kvs, kw, verify, budget=peak)
        assert _result(again) == want, name
        again.close()
        assert pool.used() == base, name


def test_inputs_that_cannot_fit_are_refused_before_upload(pkg, pool):
    """A budget below an input's device copy, or — for a compressed input — one that holds the copy but not the
    uncompressed image, is NotSupported at add_input, naming need and budget, with nothing copied to the device."""
    cfg, runs = _cfg_runs(9)
    raw = o.Sst.build(runs[0], o.TableOptions(block_size=4096))
    snappy = o.Sst.build(_phrase_runs(32, 1, 800)[0], o.TableOptions(block_size=4096, compression=1))
    img, nc = pkg.sst_uncompressed_bytes(snappy.meta_view(), snappy.data_view())
    assert nc > 0 and img > snappy.data_view().size
    # the compressed table's budget holds its device copy but only half of its uncompressed image
    for sst, budget in ((raw, raw.data_view().size // 2), (snappy, snappy.data_view().size + img // 2)):
        base = pool.used()
        job = pkg.GpuCompactionJob(device_memory_budget=budget, block_size=4096)
        with pytest.raises(pkg.YbGpuError) as ei:
            job.add_input_sst(sst.meta_view(), sst.data_view())
        assert ei.value.status_name == "NotSupported" and "device memory budget exceeded" in str(ei.value)
        assert "budget %d" % budget in str(ei.value)
        assert job.stats().h2d_bytes == 0
        job.close()
        assert pool.used() == base
    base = pool.used()
    job = pkg.GpuCompactionJob(device_memory_budget=64 << 10, block_size=4096)
    with pytest.raises(pkg.YbGpuError) as ei:
        job.add_input_kv(runs[0])
    assert ei.value.status_name == "NotSupported" and job.stats().h2d_bytes == 0
    job.close()
    assert pool.used() == base


def _oracle_kv(runs, kw):
    return o.compact([o.Sst.build(r, o.TableOptions(block_size=4096)) for r in runs],
                     o.CompactionParams(cutoff_ht=kw["cutoff_ht"]), o.TableOptions(block_size=4096))


def _files_kv(files):
    kv = []
    for data, meta in files:
        kv += o.Sst.from_bytes(bytes(meta), bytes(data)).read_all()
    return kv


@pytest.mark.parametrize("one_table", [False, True])
def test_pipelined_compactions_fit_the_budget(pkg, one_table):
    """max_subcompactions = 0 plans the ranges from the budget; ½ and ¼ of the single job's peak: the KV stream and the
    counters equal the oracle's, every range fits its share, the total peak stays within the budget. max_subcompactions
    = 1 under a budget below the single job's peak is cut into more than one range as it runs."""
    cfg, runs = _cfg_runs(21, num_rows=20000, value_len=160)
    ssts = [o.Sst.build(r, o.TableOptions(block_size=4096)) for r in runs]
    views = [(s.meta_view(), s.data_view()) for s in ssts]
    kw = dict(cutoff_ht=o.ht_from_micros(cfg.base_micros + 1500), block_size=4096)
    exp = _oracle_kv(runs, kw)
    single = gpu_single(pkg, ssts, kw)
    peak = single.stats().device_bytes_peak
    single.close()
    cases = [(0, peak // 2, 3), (0, peak // 4, 3), (1, peak * 3 // 4, 1)]
    for max_sub, budget, in_flight in cases:
        if one_table:
            data, meta, res, total = pkg.compact_files_one_table(views, max_subcompactions=max_sub, max_in_flight=in_flight,
                                                                 device_memory_budget=budget, **kw)
            kv = o.Sst.from_bytes(meta.tobytes(), data.tobytes()).read_all()
            n = res.num_ranges
        else:
            r = pkg.compact_files(views, max_subcompactions=max_sub, max_in_flight=in_flight, device_memory_budget=budget, **kw)
            kv = _files_kv(r.files())
            total, n = r.total, len(r.outputs)
            peaks = [out.stats.device_bytes_peak for out in r.outputs]
            assert max(peaks) <= budget // in_flight
            # the bytes held at once: at least one range's peak, at most all of them together
            assert max(peaks) <= total.device_bytes_peak <= sum(peaks)
            lows = [out.lower for out in r.outputs]
            assert lows == sorted(lows) and r.outputs[0].lower == b"" and r.outputs[-1].upper == b""
            assert all(a.upper == b.lower for a, b in zip(r.outputs, r.outputs[1:]))
        assert kv == exp.kv_list(), (max_sub, budget)
        assert total.num_input_records == exp.stats.num_input_records
        assert total.num_output_records == exp.stats.num_output_records
        assert 0 < total.device_bytes_peak <= budget, (total.device_bytes_peak, budget)
        assert n > 1, (max_sub, budget)


def gpu_single(pkg, ssts, kw):
    job = pkg.GpuCompactionJob(**kw)
    for s in ssts:
        job.add_input_sst(s.meta_view(), s.data_view())
    job.run()
    return job


def test_a_row_larger_than_the_budget_fails_cleanly(pkg, pool):
    """One DocKey row whose versions need more than the budget cannot be cut: the compaction fails with the budget
    message and leaves the pool as it found it."""
    runs = [r for r in w.giant_row_runs(3, n_runs=3, small_rows=0) if r]
    ssts = [o.Sst.build(r, o.TableOptions(block_size=4096)) for r in runs]
    views = [(s.meta_view(), s.data_view()) for s in ssts]
    single = gpu_single(pkg, ssts, dict(block_size=4096))
    peak = single.stats().device_bytes_peak
    single.close()
    base = pool.used()
    with pytest.raises(pkg.YbGpuError) as ei:
        pkg.compact_files(views, max_subcompactions=1, max_in_flight=1, device_memory_budget=peak // 2, block_size=4096)
    assert "device memory budget exceeded" in str(ei.value) and "no row boundary" in str(ei.value)
    assert pool.used() == base


def test_zero_subcompactions_without_a_budget_is_one_range(pkg):
    """max_subcompactions = 0 and no budget means one range, as it always has, in both pipelined calls."""
    cfg, runs = _cfg_runs(23)
    ssts = [o.Sst.build(r, o.TableOptions(block_size=4096)) for r in runs]
    views = [(s.meta_view(), s.data_view()) for s in ssts]
    kw = dict(cutoff_ht=o.ht_from_micros(cfg.base_micros + 1500), block_size=4096)
    exp = _oracle_kv(runs, kw)
    for verify in (None, True):
        r = pkg.compact_files(views, max_subcompactions=0, verify_outputs=verify, **kw)
        assert len(r.outputs) == 1 and r.outputs[0].lower == b"" and r.outputs[0].upper == b""
        assert _files_kv(r.files()) == exp.kv_list()
        assert r.total.device_bytes_peak == r.outputs[0].stats.device_bytes_peak > 0
        data, meta, res, total = pkg.compact_files_one_table(views, max_subcompactions=0, verify_outputs=verify, **kw)
        assert res.num_ranges == 1
        assert o.Sst.from_bytes(meta.tobytes(), data.tobytes()).read_all() == exp.kv_list()
