"""The kernel routes Engine::Run picks by input shape, each against the oracle and each proven by its path flag.

The bench shape (shared-prefix inputs, internal keys <= 64 B, blocks <= 32 KB, <= 24 files) runs k_ingest,
k_merge_filter and k_encode_v5; the other shapes switch kernels. Every case below compares the KV stream, every counter,
the digest, the boundaries and both output files with the oracle (test_gpu_parity.check) and asserts the route.
Internal key = user key + 8; S = record stride = roundup16(user key + 16).

| route | taken when | test |
|---|---|---|
| k_ingest, first attempt (PATH_FUSED_INGEST) | shared-prefix inputs, every block staged | test_ingest_staging_buffer_edge, test_wide_keys |
| k_ingest again at S = 80 (PATH_INGEST_RETRY) | a key longer than the probe's sample (first restart interval of some blocks) | test_ingest_stride_retry |
| fused attempt declines -> general (PATH_GENERAL_DECODE) | staged span > ING_BUF (34 304 B), > 512 entries per block, internal key > 64 B | test_ingest_staging_buffer_edge, test_more_than_512_entries_per_block, test_mixed_declines_in_one_job |
| k_decode_fast<2/3/4> (PATH_FAST_DECODE) | general path, max internal key <= 32 / 48 / 64, no key range, no HT / cotable filter | test_more_than_512_entries_per_block |
| k_decode_all<128> with filters / key ranges | the same inputs with an HT filter, cotable filters, compact_files | test_filters_and_ranges_take_decode_all |
| k_decode_all<128 / 320 / 1024> | max internal key <= 128 / 320 / 1016 | test_wide_keys, test_compact_files_long_dockeys |
| NotSupported "user keys longer than 1008 bytes" | max internal key > 1016 (table files and KV streams) | test_user_key_longer_than_1008_bytes |
| k_encode_v5 (PATH_ENCODER_V5) | 4096 + 256 * G <= 96 KB, G = ((S + 71) & ~7) + 4: user keys <= 272 B | test_wide_keys |
| k_encode_v4, no V5 (PATH_ENCODER_V4) | user keys > 272 B (internal > 280 B), both output key encodings | test_wide_keys |
| k_encode_fused (PATH_ENCODER_FUSED) | v4 route and an output block larger than the 36 KB image | test_wide_keys |
| k_records_from_kv (PATH_KV_INPUT) | KV-stream inputs, S up to 1024 | test_wide_keys_kv_inputs |
| merge-tile capacity, M -> 1 | cap = 74 368 / (S + 41) rounded down to 16: 64 records at S = 1024 | test_widest_keys_many_files |
| partition retry (PATH_PARTITION_RETRY) | largest tile > cap: M halved up to 4 times | test_partition_retry |
| NotSupported "record stride and run count too large for a merge tile" | a tile > cap at M = 1 | test_widest_keys_every_key_in_every_file |
| segment bounds in two rounds of 32 lanes, 64-cursor replays | k > 32 input files | test_many_input_files |
| 65th input file | NotSupported "too many input files" | test_65th_input_file |
| input checksums on every decode route (YBGPU_CORRUPTION) | fused, fused then general, general, stride retry | test_checksums_on_every_route |
"""
import importlib
import random

import numpy as np
import pytest

import dockv_util as dk
import oracle_py as o
import workloads as w
from test_gpu_parity import check, gpu_compact, okw, runs_to_ssts

pytestmark = pytest.mark.gpu

WIDTHS = [32, 33, 48, 49, 64, 65, 128, 129, 280, 281, 320, 321, 1016]
TWIN_PREFIXES = (15, 16, 17, 500, 1000)
TILE_TOO_SMALL = "record stride and run count too large for a merge tile"


@pytest.fixture(scope="module")
def pkg():
    m = importlib.import_module("yugabyte-db_b200")
    assert m.device_count() >= 1, "GPU tests need a CUDA device"
    return m


def has(st, *flags):
    return all(st.path_flags & f for f in flags)


def lacks(st, *flags):
    return not any(st.path_flags & f for f in flags)


def plain_kw(seq_top, bottommost=True):
    return dict(retention=False, bottommost=bottommost, last_sequence=seq_top + 1)


# ---- workloads -------------------------------------------------------------------------------------------------

def _fill(make, target):
    """make(n) builds a key with an n-byte filler (no zero bytes: the length grows by one per byte): the key of length
    exactly `target`."""
    n = target - len(make(0))
    assert n >= 0, (target, len(make(0)))
    k = make(n)
    assert len(k) == target
    return k


def plain_wide_runs(seed, width, n_runs=3, n_keys=400):
    """Plain RocksDB keys (no DocDB structure) whose longest internal key is exactly `width` bytes: ragged lengths,
    pairs that agree for their first P bytes and differ in the last one, and user keys present in several runs that
    differ only in their sequence numbers (rule A). Returns (runs, largest sequence number)."""
    rng = random.Random(seed)
    U = width - 8
    runs = [[] for _ in range(n_runs)]
    seq = 1 << 40
    keys = set()
    for i in range(n_keys):
        base = b"p%05d" % i
        keys.add(base + b"." * rng.randrange(0, U - len(base) + 1))
    keys.add(_fill(lambda n: b"z" + b"m" * n, U))
    for p in TWIN_PREFIXES:
        if p + 1 <= U:
            common = (b"t%04d" % p + bytes(rng.randrange(1, 256) for _ in range(p)))[:p]
            keys.update({common + b"\x41", common + b"\x42"})
    for uk in sorted(keys):
        for r in rng.sample(range(n_runs), 1 if rng.random() < 0.8 else min(n_runs, 3)):
            seq += 1
            runs[r].append((o.ikey(uk, seq), b"v%d" % rng.randrange(10**6) + b"w" * rng.randrange(30)))
    return [w.sort_run(r) for r in runs], seq


def docdb_wide_runs(seed, width, n_runs=3, n_rows=150, cotable=None):
    """DocDB keys whose longest internal key is exactly `width` bytes. DocKeys carry a string range component of up to
    200 bytes; a string subkey takes the rest of the length. Several versions per column, tombstones, the same user key
    in several runs (rule A), subkeys that agree for their first P key bytes and differ in the last one."""
    rng = random.Random(seed)
    U = width - 8
    runs = [[] for _ in range(n_runs)]
    seq = [(1 << 50) + (r << 30) for r in range(n_runs)]
    used = set()

    def put(uk, value, copies=1):
        assert len(uk) <= U
        if uk in used:
            return
        used.add(uk)
        for r in rng.sample(range(n_runs), copies):
            seq[r] += 1
            runs[r].append((o.ikey(uk, seq[r]), value))

    def ht():
        return (w.BASE_US + rng.randrange(12) * 10, 0, 0)

    def val():
        return dk.TOMBSTONE if rng.random() < 0.15 else dk.vstr("v%d" % rng.randrange(1000) + "x" * rng.randrange(20))

    def key(d, col, sub, h):
        return dk.sub_doc_key(d, [dk.kcol(col)] + ([sub] if sub is not None else []), ht=h)

    for row in range(n_rows):
        name = "r%05d" % row
        d0 = dk.doc_key([name], cotable=cotable)
        budget = U - len(key(d0, 1, None, ht()))
        if budget < 0:
            continue
        d = dk.doc_key([name + "." * rng.randrange(0, min(200, budget) + 1)], cotable=cotable)
        for c in range(1, rng.randrange(2, 5)):
            room = U - len(key(d, c, None, ht())) - 3
            sub = None if room < 0 or rng.random() < 0.4 else "s" * rng.randrange(0, room + 1)
            for _ in range(rng.randrange(1, 4)):
                put(key(d, c, sub, ht()), val(), 2 if rng.random() < 0.1 and n_runs > 1 else 1)
    # the longest key, and subkey twins that differ only at key byte P
    d = dk.doc_key(["zz"], cotable=cotable)
    h = (w.BASE_US + 50, 0, 0)
    room = U - len(key(d, 1, None, h))
    if room >= 3:
        put(key(d, 1, "m" * (room - 3), h), dk.vstr("longest"))
    else:
        put(_fill(lambda f: key(dk.doc_key(["zz" + "." * f], cotable=cotable), 1, None, h), U), dk.vstr("longest"))
    for p in TWIN_PREFIXES:
        dd = dk.doc_key(["tw%04d" % p], cotable=cotable)
        head = len(dd) + 2 + 1                                   # DocKey, column, 'S' of the subkey
        tail = 3 + 1 + 7                                         # the differing byte, the string's end, '#' + hybrid time
        if p >= head and p + tail <= U:
            for j in (0, 1):
                put(key(dd, 1, "q" * (p - head) + "AB"[j], h), dk.vstr("twin%d" % j))
    assert max(len(k) for r in runs for k, _ in r) == width
    return [w.sort_run(r) for r in runs if r]


def dense_runs(width, n_runs=3, n_per_run=4000, cotable=None, docdb=True):
    """Tiny entries (internal keys of exactly `width` bytes, one-byte values): far more than 512 entries in a 32 KB
    block."""
    runs = []
    seq = 1 << 40
    for r in range(n_runs):
        kvs = []
        for i in range(n_per_run):
            seq += 1
            n = r * n_per_run + i
            if docdb:
                uk = _fill(lambda f: dk.sub_doc_key(dk.doc_key(["d" + "0" * f + "%07d" % n], cotable=cotable), [dk.kcol(1)],
                                                    micros=w.BASE_US + 10 * (n % 9)), width - 8)
                v = dk.TOMBSTONE if n % 11 == 0 else b"S"
            else:
                uk = _fill(lambda f: b"d" + b"0" * f + b"%07d" % n, width - 8)
                v = b"v"
            kvs.append((o.ikey(uk, seq), v))
        runs.append(w.sort_run(kvs))
    return runs, seq


def _varint(b, p):
    r = s = 0
    while True:
        c = b[p]
        p += 1
        r |= (c & 0x7f) << s
        s += 7
        if c < 0x80:
            return r, p


def probed_keys(sst):
    """User keys of the first restart interval of every block with two or more intervals: what k_restart_probe may walk
    to guess the record stride."""
    offs, sizes = sst.block_handles()
    d = bytes(sst.data)
    out = set()
    for off, size in zip(offs, sizes):
        blk = d[int(off):int(off) + int(size)]
        nres = int.from_bytes(blk[-4:], "little")
        if nres < 2:
            continue
        ro = len(blk) - 4 - 4 * nres
        end = int.from_bytes(blk[ro + 4:ro + 8], "little")
        p, k = 0, b""
        while p < end:
            sh, p = _varint(blk, p)
            ns, p = _varint(blk, p)
            vl, p = _varint(blk, p)
            k = k[:sh] + blk[p:p + ns]
            p += ns + vl
            out.add(k[:-8])
    return out


def retry_runs(n_runs=3, n_per_run=3000):
    """Plain keys of 15 internal bytes, plus keys of 50-64 bytes that sit only in the second or a later restart interval
    of their block: the probe's sample sees 15 bytes (S = 32), k_ingest meets the long keys and runs again at S = 80."""
    rng = random.Random(5)
    runs, seq = [], 1 << 40
    for r in range(n_runs):
        kvs = []
        for i in range(n_per_run):
            seq += 1
            n = r * n_per_run + i
            kvs.append((o.ikey(b"s%06d" % n, seq), b"v" * rng.randrange(4, 24)))
            if i % 37 == 20:
                seq += 1
                kvs.append((o.ikey(b"s%06d" % n + b"~" * (35 + n % 15), seq), b"long"))
        runs.append(w.sort_run(kvs))
    for _ in range(20):
        ssts = [o.Sst.build(r, o.TableOptions(block_size=4096)) for r in runs]
        sampled = [{k for k in probed_keys(s) if len(k) > 16} for s in ssts]
        if not any(sampled):
            break
        runs = [[kv for kv in r if kv[0][:-8] not in bad] for r, bad in zip(runs, sampled)]
    else:
        raise AssertionError("long keys keep landing in sampled restart intervals")
    assert sum(1 for r in runs for k, _ in r if len(k) >= 50) >= 100
    return runs, ssts, seq


def oversize_block_runs(value_len, n_rows=30, n_runs=2):
    """One DocDB entry per input block (4 KB target, ~value_len-byte values): exact block sizes around ING_BUF."""
    runs = [[] for _ in range(n_runs)]
    rng = random.Random(value_len)
    for i in range(n_rows):
        r = i % n_runs
        uk = dk.sub_doc_key(dk.doc_key(["b%04d" % i]), [dk.kcol(1)], micros=w.BASE_US + 10 * (i % 7))
        runs[r].append((o.ikey(uk, (1 << 50) + i), b"S" + bytes(rng.randrange(1, 256) for _ in range(value_len - 1))))
    return [w.sort_run(r) for r in runs]


def max_block(ssts):
    return max(int(x) for s in ssts for x in s.block_handles()[1])


def range_outputs_kv(res):
    got = []
    for data, meta in res.files():
        got += o.Sst.from_bytes(meta.tobytes(), data.tobytes()).read_all()
    return got


# ---- a. k_ingest's declines --------------------------------------------------------------------------------------

def test_ingest_staging_buffer_edge(pkg):
    """A staged span is the block + 5-byte trailer + its 16-byte misalignment, rounded up to 16; k_ingest stages up to
    ING_BUF = 34 304 bytes. Blocks of at most 34 284 bytes are staged whatever the alignment; blocks of 34 300 or more
    never are, and the host falls back to the general kernels."""
    inside = runs_to_ssts(oversize_block_runs(34200), 4096)
    assert 34200 < max_block(inside) <= 34284
    job, _ = check(pkg, inside, block_size=32768, cutoff_ht=o.ht_from_micros(w.BASE_US + 35))
    assert has(job.stats(), pkg.PATH_FUSED_INGEST) and lacks(job.stats(), pkg.PATH_GENERAL_DECODE)
    outside = runs_to_ssts(oversize_block_runs(34320), 4096)
    assert max_block(outside) >= 34300
    job, _ = check(pkg, outside, block_size=32768, cutoff_ht=o.ht_from_micros(w.BASE_US + 35))
    assert has(job.stats(), pkg.PATH_GENERAL_DECODE) and lacks(job.stats(), pkg.PATH_FUSED_INGEST)


@pytest.mark.parametrize("width", [32, 48, 64])
def test_more_than_512_entries_per_block(pkg, width):
    """More than ING_MAXE entries in a block: the general path, which decodes internal keys of at most 32 / 48 / 64 bytes
    with k_decode_fast<2 / 3 / 4>."""
    for docdb in (True, False):
        runs, seq = dense_runs(width, docdb=docdb)
        ssts = runs_to_ssts(runs, 32768)
        assert max(len(k) for r in runs for k, _ in r) == width
        assert max(s.num_entries / len(s.block_handles()[0]) for s in ssts) > 512
        kws = [w.param_grid()[i] for i in (0, 2, 5)] if docdb else [plain_kw(seq), plain_kw(seq, False)]
        for kw in kws:
            job, _ = check(pkg, ssts, block_size=4096, **kw)
            assert has(job.stats(), pkg.PATH_GENERAL_DECODE, pkg.PATH_FAST_DECODE) and lacks(job.stats(), pkg.PATH_FUSED_INGEST)


def _uuid(t):
    return bytes([(t * 37 + j) % 251 + 1 for j in range(16)])


def test_filters_and_ranges_take_decode_all(pkg):
    """The inputs of test_more_than_512_entries_per_block with an HT filter, with cotable filters and as key ranges:
    k_decode_all<128>, never the fast kernel (it applies none of them)."""
    runs, _ = dense_runs(48)
    ssts = runs_to_ssts(runs, 32768)
    filt = [o.ht_from_micros(w.BASE_US + 45), o.HT_INVALID, o.ht_from_micros(w.BASE_US + 25)]
    job, _ = check(pkg, ssts, block_size=4096, ht_filters=filt, cutoff_ht=o.ht_from_micros(w.BASE_US + 35))
    assert has(job.stats(), pkg.PATH_GENERAL_DECODE) and lacks(job.stats(), pkg.PATH_FAST_DECODE, pkg.PATH_FUSED_INGEST)
    # cotable keys ('y' + uuid), one database filtered per file
    cot_runs, _ = dense_runs(64, cotable=_uuid(3))
    oid = int.from_bytes(_uuid(3)[12:16], "little")
    cot = [([oid], [o.ht_from_micros(w.BASE_US + 45)]), ([oid], [o.ht_from_micros(w.BASE_US + 15)]), None]
    cssts = runs_to_ssts(cot_runs, 32768)
    kw = w.param_grid()[2]
    exp = o.compact(cssts, o.CompactionParams(**kw), o.TableOptions(block_size=4096), cotable_filters=cot)
    assert exp.stats.num_input_records < sum(s.num_entries for s in cssts)          # the filters hide something
    job = pkg.GpuCompactionJob(block_size=4096, **kw)
    for s, c in zip(cssts, cot):
        job.add_input_sst(s.meta_view(), s.data_view())
        if c:
            job.set_cotable_filters(*c)
    st = job.run()
    assert job.kv_list() == exp.kv_list() and job.digest() == exp.stats.kv_hash
    assert (st.num_input_records, st.num_output_records) == (exp.stats.num_input_records, exp.stats.num_output_records)
    data, meta = job.fetch_output()
    assert (data.tobytes(), meta.tobytes()) == (exp.sst().data, exp.sst().meta)
    assert has(st, pkg.PATH_GENERAL_DECODE) and lacks(st, pkg.PATH_FAST_DECODE, pkg.PATH_FUSED_INGEST)
    # key ranges
    kw = w.param_grid()[4]
    exp = o.compact(ssts, o.CompactionParams(**kw), o.TableOptions(block_size=4096))
    res = pkg.compact_files([(s.meta_view(), s.data_view()) for s in ssts], max_subcompactions=4, max_in_flight=2, block_size=4096, **kw)
    assert len(res.outputs) >= 2
    assert range_outputs_kv(res) == exp.kv_list()
    assert res.total.num_input_records == exp.stats.num_input_records
    assert has(res.total, pkg.PATH_GENERAL_DECODE) and lacks(res.total, pkg.PATH_FAST_DECODE, pkg.PATH_FUSED_INGEST)


def test_ingest_stride_retry(pkg):
    """The probe guesses the record stride from the first restart interval of some blocks. Longer keys further into a
    block make k_ingest run once more at its widest stride; the job stays on the fused path."""
    runs, ssts, seq = retry_runs()
    for kw in (plain_kw(seq), plain_kw(seq, False)):
        job, _ = check(pkg, ssts, block_size=4096, **kw)
        st = job.stats()
        assert has(st, pkg.PATH_INGEST_RETRY, pkg.PATH_FUSED_INGEST) and lacks(st, pkg.PATH_GENERAL_DECODE)


def test_mixed_declines_in_one_job(pkg):
    """One file with more than 512 entries per block among ordinary files: k_ingest has already ingested some blocks when
    it declines the dense ones; the general path then decodes everything again."""
    dense, _ = dense_runs(40, n_runs=1, n_per_run=6000)
    runs = [r for r in w.random_docdb_runs(31, n_runs=3, n_rows=300) if r] + dense
    ssts = runs_to_ssts(runs[:3], 1024) + runs_to_ssts(runs[3:], 32768)
    for kw in [w.param_grid()[i] for i in (0, 2, 6, 9)]:
        job, _ = check(pkg, ssts, block_size=4096, filter_policy=1, filter_block_size=4096, **kw)
        assert has(job.stats(), pkg.PATH_GENERAL_DECODE) and lacks(job.stats(), pkg.PATH_FUSED_INGEST)


# ---- b. wide keys ------------------------------------------------------------------------------------------------

def _decode_route(pkg, st, width):
    if width <= 64:
        assert has(st, pkg.PATH_FUSED_INGEST) and lacks(st, pkg.PATH_GENERAL_DECODE)
    else:
        assert has(st, pkg.PATH_GENERAL_DECODE) and lacks(st, pkg.PATH_FUSED_INGEST, pkg.PATH_FAST_DECODE)


def _encoder_route(pkg, st, width):
    if width - 8 <= 272:
        assert has(st, pkg.PATH_ENCODER_V4, pkg.PATH_ENCODER_V5)
    else:
        assert has(st, pkg.PATH_ENCODER_V4) and lacks(st, pkg.PATH_ENCODER_V5)


@pytest.mark.parametrize("width", WIDTHS)
def test_wide_keys(pkg, width):
    """Longest internal key exactly on each edge of the decode kernels (32 / 48 / 64 / 128 / 320 / 1016), the merge
    tile's capacity and the v5 -> v4 assembler switch (280 / 281), plain and DocDB keys, both output key encodings,
    bloom filters, user boundary values, compressed output and output blocks larger than k_encode_v4's image."""
    runs, seq = plain_wide_runs(width, width)
    ssts = runs_to_ssts(runs, 1024)
    for enc, kw in ((1, plain_kw(seq)), (2, plain_kw(seq, False))):
        job, _ = check(pkg, ssts, block_size=2048, output_key_encoding=enc, **kw)
        _decode_route(pkg, job.stats(), width)
        _encoder_route(pkg, job.stats(), width)
    druns = docdb_wide_runs(1000 + width, width)
    dssts = runs_to_ssts(druns, 1024)
    for i, enc in ((0, 1), (2, 2), (5, 1), (9, 2)):
        job, _ = check(pkg, dssts, block_size=4096, output_key_encoding=enc, filter_policy=1, filter_block_size=1024, **w.param_grid()[i])
        _decode_route(pkg, job.stats(), width)
        _encoder_route(pkg, job.stats(), width)
    for kw in (w.param_grid()[2], w.param_grid()[4]):
        exp = o.compact(dssts, o.CompactionParams(**okw(kw)), o.TableOptions(block_size=4096))
        job = gpu_compact(pkg, dssts, block_size=4096, user_boundary_values=True, **kw)
        assert job.kv_list() == exp.kv_list()
        assert job.user_values() == exp.user_values()
    if width in (281, 1016):
        # Snappy output at the v4 width, and output blocks of 64 KB: the blocks past the 36 KB image go to k_encode_fused
        job, _ = check(pkg, dssts, block_size=4096, output_compression=1, **w.param_grid()[2])
        assert has(job.stats(), pkg.PATH_SNAPPY_OUTPUT)
        big = runs_to_ssts(docdb_wide_runs(4000 + width, width, n_rows=600), 4096)
        for enc in (1, 2):
            job, _ = check(pkg, big, block_size=65536, output_key_encoding=enc, **w.param_grid()[0])
            assert job.stats().num_output_data_blocks >= 2, enc
            assert has(job.stats(), pkg.PATH_ENCODER_V4, pkg.PATH_ENCODER_FUSED) and lacks(job.stats(), pkg.PATH_ENCODER_V5), enc


@pytest.mark.parametrize("width", WIDTHS)
def test_wide_keys_kv_inputs(pkg, width):
    """The same widths as KV-stream inputs (k_records_from_kv at strides up to 1024)."""
    for docdb in (False, True):
        if docdb:
            runs = docdb_wide_runs(2000 + width, width)
            kws = [w.param_grid()[2], w.param_grid()[5]]
        else:
            runs, seq = plain_wide_runs(3000 + width, width)
            kws = [plain_kw(seq), plain_kw(seq, False)]
        ssts = runs_to_ssts(runs, 1024)
        for kw in kws:
            exp = o.compact(ssts, o.CompactionParams(**kw), o.TableOptions(block_size=2048))
            job = pkg.GpuCompactionJob(block_size=2048, **kw)
            for r in runs:
                job.add_input_kv(r)
            st = job.run()
            assert has(st, pkg.PATH_KV_INPUT)
            _encoder_route(pkg, st, width)
            assert job.kv_list() == exp.kv_list() and job.digest() == exp.stats.kv_hash
            assert (st.num_input_records, st.num_output_records) == (exp.stats.num_input_records, exp.stats.num_output_records)
            assert st.num_record_drop_hidden == exp.stats.num_dropped_hidden
            data, meta = job.fetch_output()
            ref = exp.sst()
            assert (data.tobytes(), meta.tobytes()) == ((ref.data, ref.meta) if ref is not None else (b"", b""))


def test_user_key_longer_than_1008_bytes(pkg):
    runs, seq = plain_wide_runs(7, 1017, n_keys=50)
    ssts = runs_to_ssts(runs, 4096)
    job = pkg.GpuCompactionJob(**plain_kw(seq))
    for s in ssts:
        job.add_input_sst(s.meta_view(), s.data_view())
    with pytest.raises(pkg.YbGpuError) as e:
        job.run()
    assert e.value.status_name == "NotSupported" and "user keys longer than 1008 bytes" in str(e.value)
    job = pkg.GpuCompactionJob(**plain_kw(seq))
    for r in runs:
        job.add_input_kv(r)
    with pytest.raises(pkg.YbGpuError) as e:
        job.run()
    assert e.value.status_name == "NotSupported" and "user keys longer than 1008 bytes" in str(e.value)


def _long_dockey_runs(seed, dockey_len, n_runs=3, n_rows=200, pad_first=False):
    """DocKeys of dockey_len[0]..dockey_len[1] bytes, three columns, one with a long string subkey. pad_first: the DocKeys
    share their padding and differ only after it, so that even the shortest index separators are that long."""
    rng = random.Random(seed)
    runs = [[] for _ in range(n_runs)]
    seq = [(1 << 50) + (r << 30) for r in range(n_runs)]
    for row in range(n_rows):
        n = dockey_len[0] + rng.randrange(dockey_len[1] - dockey_len[0] + 1)
        head = "-" * 260 if pad_first else ""
        d = _fill(lambda f: dk.doc_key([head + "k%04d" % row + "-" * f]), n)
        for c in range(1, 4):
            for v in range(rng.randrange(1, 4)):
                sub = [dk.kcol(c)] + (["e" * rng.randrange(20, 90)] if c == 3 else [])
                uk = dk.sub_doc_key(d, sub, micros=w.BASE_US + 10 * v + 10 * rng.randrange(3))
                r = rng.randrange(n_runs)
                seq[r] += 1
                runs[r].append((o.ikey(uk, seq[r]), dk.TOMBSTONE if rng.random() < 0.1 else dk.vstr("x" * rng.randrange(40))))
    return [w.sort_run(r) for r in runs]


def test_compact_files_long_dockeys(pkg):
    """Key ranges over DocKeys of 100-200 bytes with long subkeys (k_decode_all<320> with a key range), and over DocKeys
    of 256-400 bytes: splitters are cut from the shortened index separators, which still fit YBGPU_MAX_SPLITTER_LEN when
    the DocKeys differ early, and do not when they share a 260-byte head: no splitter inside the keys, all of the
    compaction is one range."""
    for dockeys, shortest, longest in (((100, 200), 128, 320), ((256, 400), 320, 1016)):
        ssts = runs_to_ssts(_long_dockey_runs(1, dockeys), 2048)
        assert shortest < max(len(k) for s in ssts for k, _ in s.read_all()) <= longest
        for kw in (w.param_grid()[2], w.param_grid()[7]):
            exp = o.compact(ssts, o.CompactionParams(**kw), o.TableOptions(block_size=4096))
            res = pkg.compact_files([(s.meta_view(), s.data_view()) for s in ssts], max_subcompactions=4, max_in_flight=2, block_size=4096, **kw)
            assert len(res.outputs) >= 2
            assert range_outputs_kv(res) == exp.kv_list()
            assert (res.total.num_input_records, res.total.num_output_records) == (exp.stats.num_input_records, exp.stats.num_output_records)
            assert has(res.total, pkg.PATH_GENERAL_DECODE) and lacks(res.total, pkg.PATH_FUSED_INGEST, pkg.PATH_FAST_DECODE)
    ssts = runs_to_ssts(_long_dockey_runs(2, (280, 400), pad_first=True), 2048)
    kw = w.param_grid()[2]
    exp = o.compact(ssts, o.CompactionParams(**kw), o.TableOptions(block_size=4096))
    res = pkg.compact_files([(s.meta_view(), s.data_view()) for s in ssts], max_subcompactions=4, max_in_flight=2, block_size=4096, **kw)
    # the one splitter left is the last file's short successor of its last key ("T"): past every key, its range is empty
    assert len(res.files()) == 1
    data, meta = res.files()[0]
    assert (data.tobytes(), meta.tobytes()) == (exp.sst().data, exp.sst().meta)
    assert res.total.num_output_records == exp.stats.num_output_records


# ---- c. many input files -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", [16, 17, 32, 33, 64])
def test_many_input_files(pkg, k):
    """k files around the two-level rank search (<= 16 runs), the second round of 32 lanes of the segment bounds
    (> 32 runs) and MAX_RUNS = 64; rows larger than a tile spread over all runs (replays with more than 32 cursors)."""
    runs = w.random_docdb_runs(700 + k, n_runs=k, n_rows=12 * k)
    ssts = runs_to_ssts(runs, 1024)
    assert len(ssts) == k
    for kw in w.param_grid():
        check(pkg, ssts, block_size=2048, **kw)
    runs = w.random_cotable_runs(710 + k, n_runs=k, n_tables=4, rows_per_table=6 * k, colocated=k % 2 == 0)
    ssts = runs_to_ssts(runs, 1024)
    assert len(ssts) == k
    for kw in w.param_grid()[:4]:
        check(pkg, ssts, block_size=2048, **kw)
    runs = w.giant_row_runs(720 + k, n_runs=k, cols=150, versions=12, collection=800, colocated=k % 2 == 1)
    ssts = runs_to_ssts(runs, 4096)
    assert len(ssts) == k
    for kw in (w.param_grid()[2], w.param_grid()[4]):
        job, _ = check(pkg, ssts, block_size=4096, **kw)
        assert job.stats().tiles_inside_rows > 0
    if k == 64:
        ssts = runs_to_ssts(w.random_docdb_runs(730, n_runs=64, n_rows=800), 1024)
        kw = w.param_grid()[2]
        exp = o.compact(ssts, o.CompactionParams(**kw), o.TableOptions(block_size=4096))
        res = pkg.compact_files([(s.meta_view(), s.data_view()) for s in ssts], max_subcompactions=5, max_in_flight=2, block_size=4096, **kw)
        assert len(res.outputs) >= 3
        assert range_outputs_kv(res) == exp.kv_list()
        assert (res.total.num_input_records, res.total.num_output_records) == (exp.stats.num_input_records, exp.stats.num_output_records)


def test_65th_input_file(pkg):
    ssts = runs_to_ssts(w.random_docdb_runs(740, n_runs=65, n_rows=400), 1024)
    assert len(ssts) == 65
    job = pkg.GpuCompactionJob()
    for s in ssts[:64]:
        job.add_input_sst(s.meta_view(), s.data_view())
    with pytest.raises(pkg.YbGpuError) as e:
        job.add_input_sst(ssts[64].meta_view(), ssts[64].data_view())
    assert e.value.status_name == "NotSupported" and "too many input files" in str(e.value)


# ---- d. tiles at the edge ------------------------------------------------------------------------------------------

def _check_or_refused(pkg, ssts, **kw):
    """'parity' (every check of test_gpu_parity.check holds), or 'refused' with exactly the NotSupported status of a
    partition whose tiles stay too large at M = 1. Any other status fails."""
    try:
        check(pkg, ssts, **kw)
    except pkg.YbGpuError as e:
        assert e.status_name == "NotSupported" and TILE_TOO_SMALL in str(e), str(e)
        return "refused"
    return "parity"


@pytest.mark.parametrize("k", [8, 16, 32, 64])
def test_widest_keys_many_files(pkg, k):
    """1016-byte internal keys (S = 1024: 64 records per merge tile, sample stride M = 2 at 8 files and 1 above) in k
    files of ordinary shape (ragged plain keys, DocDB rows): oracle parity."""
    runs, seq = plain_wide_runs(800 + k, 1016, n_runs=k, n_keys=30 * k)
    ssts = runs_to_ssts(runs, 4096)
    assert len(ssts) == k
    assert _check_or_refused(pkg, ssts, block_size=4096, **plain_kw(seq)) == "parity"
    dssts = runs_to_ssts(docdb_wide_runs(810 + k, 1016, n_runs=k, n_rows=20 * k), 4096)
    assert _check_or_refused(pkg, dssts, block_size=4096, **w.param_grid()[2]) == "parity"


@pytest.mark.parametrize("k,outcome", [(17, "parity"), (33, "refused"), (64, "refused")])
def test_widest_keys_every_key_in_every_file(pkg, k, outcome):
    """1008-byte user keys, two versions of every key in every one of k files: a row group of 2k records whose first
    sample in every file splits at its start. At M = 1 a tile from there holds up to H + 2k = 41 + 2k records; past 64
    the partition cannot shrink it and the job is refused (DESIGN.md section 8.3). The outcome is pinned per k."""
    runs = [[] for _ in range(k)]
    seq = 1 << 40
    for g in range(40):
        for _ in range(2):
            for r in range(k):
                seq += 1
                runs[r].append((o.ikey(b"g%04d" % g + b"." * 1003, seq), b"v%d" % seq))
    ssts = runs_to_ssts([w.sort_run(r) for r in runs], 4096)
    assert _check_or_refused(pkg, ssts, block_size=4096, **plain_kw(seq)) == outcome


@pytest.mark.parametrize("k,n_before", [(2, 1267), (4, 651)])
def test_partition_retry(pkg, k, n_before):
    """3 000 versions of one user key spread over k runs (plain mode: a row group is one user key), behind n_before small
    keys. At S = 32 a tile holds 1 008 records, H = 655 and M = 353 / k. The first sample of every run inside the hot key
    splits at the key's start, the next one M records later is the first to split inside it: the tile from the key's start
    is about H + (2M - 1)k records (1 056 and 1 039 records here, the n_before values that overflow most), more than a
    tile. The partition is repeated with M halved, and the result still matches the oracle."""
    rng = random.Random(1)
    runs = [[] for _ in range(k)]
    seq = 1 << 40
    for j in range(n_before):
        seq += 1
        runs[j % k].append((o.ikey(b"a%05d" % j, seq), b"x" * (j % 30)))
    for i in range(3000):
        seq += 1
        runs[rng.randrange(k)].append((o.ikey(b"hot-key", seq), b"v%d" % i))
    for j in range(300):
        seq += 1
        runs[j % k].append((o.ikey(b"z%05d" % j, seq), b"y" * (j % 20)))
    ssts = runs_to_ssts([w.sort_run(r) for r in runs], 4096)
    for kw in (plain_kw(seq), plain_kw(seq, False)):
        job, _ = check(pkg, ssts, block_size=4096, **kw)
        assert has(job.stats(), pkg.PATH_PARTITION_RETRY)


# ---- e. checksums on every route -----------------------------------------------------------------------------------

def _flip_crc(sst, block):
    offs, sizes = sst.block_handles()
    d = np.array(sst.data_view(), copy=True)
    d[int(offs[block]) + int(sizes[block]) + 1] ^= 0xff          # the trailer: type byte, then the masked CRC32C
    return d


def _run_files(pkg, files, **kw):
    job = pkg.GpuCompactionJob(**kw)
    for meta, data in files:
        job.add_input_sst(meta, data)
    job.run()
    return job


def test_checksums_on_every_route(pkg):
    """One damaged stored CRC in an input that takes each decode route is Corruption; with verify_checksums=False the
    same job completes and matches the oracle. On the fallback route the damaged block is one k_ingest declined to stage
    (larger than ING_BUF), so only the general path's k_crc_blocks can see it."""
    kw = w.param_grid()[2]
    fused = runs_to_ssts(docdb_wide_runs(50, 64, n_rows=300), 1024)
    big = runs_to_ssts(oversize_block_runs(34320, n_rows=12, n_runs=1), 4096)
    mixed = fused[:2] + big
    tsp = [o.Sst.build(s.read_all(), o.TableOptions(block_size=1024, key_encoding=2)) for s in fused]
    _, retry, seq = retry_runs(n_runs=2, n_per_run=2000)
    cases = [("fused", fused, 1, 3, kw, pkg.PATH_FUSED_INGEST),
             ("fused then general", mixed, 2, 5, kw, pkg.PATH_GENERAL_DECODE),
             ("general", tsp, 0, 2, kw, pkg.PATH_GENERAL_DECODE),
             ("stride retry", retry, 1, 4, plain_kw(seq), pkg.PATH_INGEST_RETRY)]
    assert max_block(big) >= 34300
    for name, ssts, f, b, ckw, route in cases:
        exp = o.compact(ssts, o.CompactionParams(**ckw), o.TableOptions(block_size=4096))
        files = [(s.meta_view(), _flip_crc(s, b) if i == f else s.data_view()) for i, s in enumerate(ssts)]
        with pytest.raises(pkg.YbGpuError) as e:
            _run_files(pkg, files, block_size=4096, **ckw)
        assert e.value.status_name == "Corruption", name
        job = _run_files(pkg, files, block_size=4096, verify_checksums=False, **ckw)
        assert has(job.stats(), route), name
        assert job.kv_list() == exp.kv_list(), name
        data, meta = job.fetch_output()
        assert (data.tobytes(), meta.tobytes()) == (exp.sst().data, exp.sst().meta), name
