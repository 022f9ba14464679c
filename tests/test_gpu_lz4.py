"""kLZ4Compression on the GPU: LZ4 input blocks uncompressed in the same pass as raw and Snappy blocks (lz4_warp_decode),
and LZ4 output blocks written by k_lz4_compress. KV streams, counters and digests against the oracle run over the
uncompressed twins of the inputs; LZ4 data files against the reference restatement of the encoder applied to the
oracle's output (tests/lz4_util.py), metadata files against the engine's host writer, block contents against liblz4 and
pyarrow's lz4_raw."""
import numpy as np
import pytest

import lz4_util as z
import oracle_py as o
import workloads as w
from test_gpu_parity import _phrase_runs, _stored_types, gpu_compact, okw, pkg  # noqa: F401 (pkg: the fixture)

pytestmark = pytest.mark.gpu

LIB = z.liblz4()
PA = z.pyarrow_lz4()


def check_lz4(pkg, tables, twins, block_size=4096, output_compression=0, **kw):
    """check() of test_gpu_parity for inputs the oracle does not read: the GPU job runs over `tables`, the oracle over
    their uncompressed `twins`. KV stream, counters, digest and boundaries equal; the output files equal the oracle's
    (output_compression 0) or, for LZ4 output, the data file equals the reference restatement's LZ4 re-storage of the
    oracle's data file and the metadata file equals the engine's host writer's for the same entries."""
    enc, filt, fbs = kw.get("output_key_encoding", 1), kw.get("filter_policy", 0), kw.get("filter_block_size", 65536)
    exp = o.compact(twins, o.CompactionParams(**okw(kw)), o.TableOptions(block_size=block_size, key_encoding=enc, filter_policy=filt,
                                                                          filter_block_size=fbs))
    job = gpu_compact(pkg, tables, block_size=block_size, output_compression=output_compression, **kw)
    st, es, ekv = job.stats(), exp.stats, exp.kv_list()
    assert job.boundaries() == ((ekv[0][0], ekv[-1][0]) if ekv else (b"", b""))
    assert job.kv_list() == ekv and job.digest() == es.kv_hash
    assert (st.num_input_records, st.num_output_records, st.num_record_drop_hidden, st.num_record_drop_obsolete, st.num_record_drop_feed) == \
        (es.num_input_records, es.num_output_records, es.num_dropped_hidden, es.num_dropped_obsolete, es.num_dropped_feed)
    assert (st.total_input_raw_key_bytes, st.total_input_raw_value_bytes, st.total_output_raw_key_bytes, st.total_output_raw_value_bytes) == \
        (es.in_key_bytes, es.in_val_bytes, es.out_key_bytes, es.out_val_bytes)
    data, meta = (x.tobytes() for x in job.fetch_output())
    ref = exp.sst()
    if output_compression == 0:
        assert data == ref.data and meta == ref.meta
    else:
        assert data == z.reference_lz4_data_file(ref)[0]
        assert meta == z.host_lz4_table(pkg, ekv, block_size=block_size, key_encoding=enc, filter_policy=filt, filter_block_size=fbs).meta
    return job, exp


@pytest.mark.parametrize("seed", range(4))
def test_lz4_compressed_inputs(pkg, seed):
    """LZ4 input tables (files that mix LZ4 and raw blocks): checksums of the stored bytes, the blocks uncompressed on the
    GPU, then the same compaction as over raw inputs — KV stream, counters, digest and both output files equal the
    oracle's; PATH_LZ4 exactly when a block was stored compressed. Pipelined ranges agree; a flipped bit and a malformed
    stream under a valid checksum are Corruption."""
    if seed < 2:
        runs = w.random_docdb_runs(700 + seed, n_runs=3, n_rows=150 + 100 * seed)
        kws = [w.param_grid()[i] for i in (0, 2, 6)]
    else:
        cfg = o.GenConfig(seed=70 + seed, num_rows=4000, cols=2, versions=3, num_files=3, value_len=24 if seed == 2 else 200, tombstone_per_1024=50)
        runs = [s.read_all() for s in o.Sst.generate_all(cfg, o.TableOptions(block_size=4096))]
        if seed == 3:
            runs = [[(k, v[:1] + (k[-12:-8] * 50)[:len(v) - 1]) if v[:1] == b"S" and (i // 150) % 2 else (k, v) for i, (k, v) in enumerate(r)] for r in runs]
        kws = [dict(cutoff_ht=o.ht_from_micros(cfg.base_micros + 1500))]
    ibs = 2048 if seed < 2 else 8192
    ssts = [z.host_lz4_table(pkg, r, block_size=ibs) for r in runs if r]
    plain = [o.Sst.build(r, o.TableOptions(block_size=ibs)) for r in runs if r]
    any_lz4 = any(4 in s.types(pkg) for s in ssts)
    assert any_lz4 and (seed != 3 or all(0 in s.types(pkg) for s in ssts))
    for kw in kws:
        job, _ = check_lz4(pkg, ssts, plain, block_size=4096, filter_policy=1, filter_block_size=4096, **kw)
        flags = job.stats().path_flags
        assert bool(flags & pkg.PATH_LZ4) == any_lz4 and not flags & pkg.PATH_SNAPPY
    assert not gpu_compact(pkg, plain, block_size=4096, **kws[0]).stats().path_flags & pkg.PATH_LZ4
    exp = o.compact(plain, o.CompactionParams(**kws[0]), o.TableOptions(block_size=4096))
    res = pkg.compact_files([(s.meta_view(), s.data_view()) for s in ssts], max_subcompactions=3, max_in_flight=2, block_size=4096, **kws[0])
    got = []
    for data, meta in res.files():
        got += o.Sst.from_bytes(meta.tobytes(), data.tobytes()).read_all()
    assert got == exp.kv_list()
    # a flipped bit: checksum error
    bad = bytearray(ssts[0].data)
    bad[len(bad) // 2] ^= 0x10
    job = pkg.GpuCompactionJob(block_size=4096)
    job.add_input_sst(ssts[0].meta_view(), np.frombuffer(bytes(bad), np.uint8))
    with pytest.raises(pkg.YbGpuError) as e:
        job.run()
    assert e.value.status_name == "Corruption"
    # a malformed stream under a valid (recomputed) checksum: the decoder's own rejection
    offs, sizes = ssts[0].block_handles(pkg)
    d = bytearray(ssts[0].data)
    a, b = next((int(a), int(b)) for a, b in zip(offs, sizes) if d[int(a) + int(b)] == 4)
    n, body = z.strip_preamble(bytes(d[a:a + b]))
    stored = z.varint(n + 1) + body                                  # one byte more announced than the stream holds
    assert len(stored) == b
    d[a:a + b + 5] = stored + z._trailer(stored, 4)
    with pytest.raises(ValueError):
        z.reference_uncompress(stored)
    job = pkg.GpuCompactionJob(block_size=4096)
    job.add_input_sst(ssts[0].meta_view(), np.frombuffer(bytes(d), np.uint8))
    with pytest.raises(pkg.YbGpuError) as e:
        job.run()
    assert e.value.status_name == "Corruption"


@pytest.mark.skipif(LIB is None or not hasattr(LIB, "LZ4_compress_HC"), reason="liblz4.so.1 with LZ4_compress_HC is needed")
def test_library_written_and_mixed_inputs(pkg):
    """Tables whose LZ4 blocks liblz4 wrote (default, and HC stored as kLZ4HCCompression) compact to the output of their
    raw twins; one job over raw, Snappy, LZ4 and LZ4HC tables sets PATH_SNAPPY and PATH_LZ4 and equals the oracle."""
    runs = _phrase_runs(910, 4, 600)
    kw = w.param_grid()[0]
    raw = [o.Sst.build(r, o.TableOptions(block_size=2048)) for r in runs]
    ref = gpu_compact(pkg, raw, block_size=4096, **kw)
    rdata, rmeta = (x.tobytes() for x in ref.fetch_output())
    for mode, t in (("default", 4), ("hc", 5)):
        tabs = []
        for r in runs:
            meta, data, n = z.library_table(pkg, r, LIB, mode, t, block_size=2048)
            assert n > 0
            tabs.append(z.Table(meta, data))
        job = gpu_compact(pkg, tabs, block_size=4096, **kw)
        assert job.stats().path_flags & pkg.PATH_LZ4
        data, meta = job.fetch_output()
        assert data.tobytes() == rdata and meta.tobytes() == rmeta and job.kv_list() == ref.kv_list()
    m5, d5, _ = z.library_table(pkg, runs[3], LIB, "hc", 5, block_size=2048)
    mixed = [raw[0], o.Sst.build(runs[1], o.TableOptions(block_size=2048, compression=1)),
             z.host_lz4_table(pkg, runs[2], block_size=2048), z.Table(m5, d5)]
    job, _ = check_lz4(pkg, mixed, raw, block_size=4096, filter_policy=1, filter_block_size=4096, **kw)
    assert job.stats().path_flags & pkg.PATH_SNAPPY and job.stats().path_flags & pkg.PATH_LZ4


@pytest.mark.parametrize("seed", range(4))
def test_lz4_compressed_output(pkg, seed):
    """output_compression = 4: every assembled data block goes through k_lz4_compress and is stored as kLZ4Compression when
    that saves 12.5 %; files byte-identical to the oracle's; each stored LZ4 block, decoded by liblz4 and pyarrow, is the
    uncompressed twin's block at that index; verify_blocks finds no bad block; the table is a valid next input; the
    pipelined one-table compaction writes LZ4 too."""
    if seed == 0:
        runs, bs, enc, kws = _phrase_runs(920, 3, 300), 1024, 1, [w.param_grid()[i] for i in (0, 2, 6)]
    elif seed == 1:
        runs, bs, enc, kws = _phrase_runs(921, 4, 1500, random_every=120), 4096, 2, [w.param_grid()[0]]
    elif seed == 2:
        runs, bs, enc, kws = _phrase_runs(922, 3, 4000, vmax=400, random_every=700), 32768, 1, [w.param_grid()[2]]
    else:
        runs = _phrase_runs(923, 2, 60)
        big = [(k, b"S" + (bytes(range(256)) * 700)[:150000 + 7 * i] if i % 9 == 4 and v[:1] == b"S" else
                (b"S" + b"\0" * (3000 + i) if i % 9 == 7 and v[:1] == b"S" else v)) for i, (k, v) in enumerate(runs[0])]
        runs, bs, enc, kws = [big, runs[1]], 2048, 2, [w.param_grid()[0]]
    ssts = [z.host_lz4_table(pkg, r, block_size=bs) for r in runs if r]
    twins = [o.Sst.build(r, o.TableOptions(block_size=bs)) for r in runs if r]
    for kw in kws:
        job, exp = check_lz4(pkg, ssts, twins, block_size=bs, output_key_encoding=enc, filter_policy=1, filter_block_size=4096,
                             output_compression=4, **kw)
        assert job.stats().path_flags & pkg.PATH_LZ4_OUTPUT and not job.stats().path_flags & pkg.PATH_SNAPPY_OUTPUT
        data, meta = (x.tobytes() for x in job.fetch_output())
        types, off, sz = _stored_types(data, meta, pkg)
        plain = gpu_compact(pkg, ssts, block_size=bs, output_key_encoding=enc, filter_policy=1, filter_block_size=4096, **kw)
        pdata, pmeta = (x.tobytes() for x in plain.fetch_output())
        ptypes, poff, psz = _stored_types(pdata, pmeta, pkg)
        assert len(types) == len(ptypes) and set(ptypes) == {0} and 4 in types and set(types) <= {0, 4}
        if seed in (1, 2):
            assert 0 in types
        for t, a, b, pa_, pb in zip(types, off, sz, poff, psz):
            stored = data[int(a):int(a) + int(b)]
            want = pdata[int(pa_):int(pa_) + int(pb)]
            if t == 0:
                assert stored == want
                continue
            assert len(stored) < len(want) - len(want) // 8
            n, body = z.strip_preamble(stored)
            assert n == len(want) and z.reference_uncompress(stored) == want
            if LIB:
                assert z.lib_decompress(LIB, body, n) == want
            if PA:
                assert PA.decompress(body, decompressed_size=n, codec="lz4_raw").to_pybytes() == want
        assert pkg.sst_verify_blocks(np.frombuffer(meta, np.uint8), np.frombuffer(data, np.uint8)) == (len(types), 0)
    # the (last) LZ4 table is a valid input of the next compaction: the same entries as the next compaction of its raw
    # twin, exp.sst()
    kw = kws[0]
    again = gpu_compact(pkg, [z.Table(meta, data)], block_size=bs, **kw)
    assert again.stats().path_flags & pkg.PATH_LZ4
    assert again.kv_list() == o.compact([exp.sst()], o.CompactionParams(**okw(kw)), o.TableOptions(block_size=bs)).kv_list()
    exp = o.compact(twins, o.CompactionParams(**okw(kw)), o.TableOptions(block_size=bs, key_encoding=enc))
    nxt = o.compact([exp.sst()], o.CompactionParams(**okw(kw)), o.TableOptions(block_size=bs)).kv_list()
    # pipelined key ranges with LZ4 output assemble into one LZ4 table holding the single job's entries
    files = [(s.meta_view(), s.data_view()) for s in ssts]
    d1, m1, res, total = pkg.compact_files_one_table(files, max_subcompactions=4, max_in_flight=2, block_size=bs, output_key_encoding=enc,
                                                     filter_policy=1, filter_block_size=4096, output_compression=4, **kw)
    d1, m1 = d1.tobytes(), m1.tobytes()
    assert total.path_flags & pkg.PATH_LZ4_OUTPUT and 4 in _stored_types(d1, m1, pkg)[0]
    assert pkg.sst_verify_blocks(z.np_u8(m1), z.np_u8(d1))[1] == 0
    assert gpu_compact(pkg, [z.Table(m1, d1)], block_size=bs, **kw).kv_list() == nxt


def test_unsupported_output_compression(pkg):
    for c in (2, 5, 7):
        with pytest.raises(pkg.YbGpuError) as e:
            pkg.GpuCompactionJob(output_compression=c)
        assert e.value.status_name == "NotSupported"


def test_raw_lz4_raw_round_trip_2m_entries(pkg):
    """A ~2 M-entry generated compaction, raw -> LZ4 and then LZ4 -> raw, gives the KV digest of raw -> raw."""
    cfg = pkg.GenConfig(seed=31, num_rows=500000, cols=2, versions=2, num_files=4, value_len=16, tombstone_per_1024=20)
    gens = pkg.generate_ssts(cfg, block_size=32768)
    files = [(g.meta_view(), g.data_view()) for g in gens]

    def run(inputs, comp):
        job = pkg.GpuCompactionJob(block_size=32768, retain_delete_markers=True, output_compression=comp)
        for m, d in inputs:
            job.add_input_sst(m, d)
        job.run()
        return job

    direct = run(files, 0)
    assert direct.stats().num_input_records >= 1_000_000
    lz = run(files, 4)
    assert lz.stats().path_flags & pkg.PATH_LZ4_OUTPUT
    ldata, lmeta = lz.fetch_output()
    ldata, lmeta = ldata.copy(), lmeta.copy()
    back = run([(lmeta, ldata)], 0)
    assert back.stats().path_flags & pkg.PATH_LZ4
    assert back.digest() == direct.digest() == lz.digest()
