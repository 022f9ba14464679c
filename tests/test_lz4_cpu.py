"""kLZ4Compression blocks without a GPU: the reference restatement of the engine's LZ4 encoder (tests/lz4_util.py) against
two independent LZ4 implementations (the system's liblz4 and pyarrow's lz4_raw); the decoders as a safety boundary (they
never accept what liblz4 rejects); the LZ4 kernels' SOURCE on emulated warps (tests/host_harness/lz4_emu.cc); the host
writer, reader and ABI entry points."""
import importlib
import random

import numpy as np
import pytest

import lz4_util as z
import oracle_py as o

LIB = z.liblz4()
PA = z.pyarrow_lz4()


@pytest.fixture(scope="module")
def pkg():
    import __graft_entry__ as g
    g.build()
    return importlib.import_module("yugabyte-db_b200")


def _inputs():
    rng = random.Random(5)
    words = [bytes(rng.randrange(32, 127) for _ in range(rng.randrange(2, 14))) for _ in range(40)]
    phrase = b" ".join(rng.choice(words) for _ in range(40000))
    out = [("empty", b"")]
    out += [("short%d" % k, bytes(rng.randrange(256) for _ in range(k))) for k in range(1, 13)]
    out += [("run%d" % k, b"a" * k) for k in (12, 13, 17)]
    out += [("zeros", bytes(100000)), ("random", bytes(rng.randrange(256) for _ in range(20000))), ("phrases", phrase)]
    for period in (1, 2, 3, 31, 32, 33):
        pat = bytes(rng.randrange(256) for _ in range(period))
        out.append(("period%d" % period, (pat * (70000 // period + 1))[:70000]))
    for n in (65535, 65536, 65537):
        out.append(("frag%d" % n, phrase[:n]))
    out += [("150k", (bytes(range(256)) * 700)[:150000]), ("1m", (phrase * 4)[:1 << 20])]
    return out


def test_reference_codec_round_trip_and_library_cross_check():
    """The reference restatement's streams decode by liblz4's LZ4_decompress_safe, by pyarrow and by the strict reference
    decoder to the input; the reference decoder reads liblz4's own streams (default, fast at several accelerations, HC
    where exported)."""
    for name, raw in _inputs():
        c = z.reference_compress(raw)
        n, body = z.strip_preamble(c)
        assert n == len(raw), name
        assert z.reference_uncompress(c) == raw, name
        if LIB:
            assert z.lib_decompress(LIB, body, len(raw)) == raw, name
            pre = z.varint(len(raw))
            for mode, accel in [("default", 1), ("fast", 1), ("fast", 8), ("fast", 65)] + ([("hc", 9), ("hc", 12)] if hasattr(LIB, "LZ4_compress_HC") else []):
                assert z.reference_uncompress(pre + z.lib_compress(LIB, raw, mode, accel)) == raw, (name, mode, accel)
        if PA and raw:
            assert PA.decompress(body, decompressed_size=len(raw), codec="lz4_raw").to_pybytes() == raw, name
    if not LIB and not PA:
        pytest.skip("neither liblz4.so.1 nor pyarrow's lz4_raw is available: only the reference round trip ran")


def _hand_made():
    """(stream incl. preamble, what it is) — every one malformed."""
    lit = lambda b: bytes([len(b) << 4]) + b                                           # noqa: E731 (len < 15)
    good_head = bytes([0x40]) + b"abcd"                                                 # 4 literals, then a match follows
    return [
        (z.varint(5), "no token"),
        (z.varint(20) + bytes([0xf0]), "truncated literal length"),
        (z.varint(20) + bytes([0xf0, 0xff]), "truncated literal length run"),
        (z.varint(5) + bytes([0x50]) + b"abc", "truncated literal"),
        (z.varint(30) + good_head + bytes([4]), "truncated offset"),
        (z.varint(30) + good_head + bytes([0, 0]) + lit(b"x" * 10), "offset 0"),
        (z.varint(30) + good_head + bytes([5, 0]) + lit(b"x" * 10), "offset before the output start"),
        (z.varint(30) + bytes([0x4f]) + b"abcd" + bytes([1, 0]), "truncated match length"),
        (z.varint(4) + lit(b"abcde"), "output longer than announced"),
        (z.varint(6) + lit(b"abcde"), "output shorter than announced"),
        (z.varint(26) + bytes([0xc4]) + b"x" * 12 + bytes([1, 0]) + lit(b"y" * 6), "a valid stream (control): ok?"),
        (z.varint(20) + bytes([0xc0]) + b"x" * 12 + bytes([1, 0]), "a stream ending in a match"),
        (z.varint(20) + bytes([0xc4]) + b"x" * 12 + bytes([1, 0]) + lit(b"y" * 0), "the last sequence empty after a match"),
        (z.varint(20) + bytes([0xc0]) + b"x" * 12 + bytes([1, 0]) + lit(b"y" * 4), "a match inside the last 5 bytes"),
        (z.varint(17) + lit(b"x" * 6) + bytes([1, 0]) + lit(b"y" * 7), "a match starting within the last 12 bytes"),
    ]


def _agree(stream):
    """The reference decoder accepts only what liblz4 accepts (capacity = the announced length), and then to the same
    bytes. Returns the reference's verdict."""
    try:
        got = z.reference_uncompress(stream)
    except ValueError:
        got = None
    if LIB:
        n, body = z.strip_preamble(stream) if stream and not all(b & 128 for b in stream) else (0, None)
        lib = z.lib_decompress(LIB, body, n) if body is not None else None
        if lib is not None and len(lib) != n:
            lib = None                                                                  # a short output is not the block
        if got is not None:
            assert lib == got, stream
    return got


def test_reference_decoder_rejections_agree_with_liblz4():
    """Hand-made malformed streams are rejected; a few thousand seeded single-byte mutations of valid streams: whatever
    liblz4 rejects the reference decoder rejects, whatever both accept decodes to the same bytes. (The engine's decoders
    are held to this reference below.)"""
    for s, what in _hand_made():
        got = _agree(s)
        if what.endswith("ok?"):
            assert got == b"x" * 12 + b"x" * 8 + b"y" * 6, what                          # the control: a valid stream
        else:
            assert got is None, what
    rng = random.Random(77)
    srcs = [raw for _, raw in _inputs() if 0 < len(raw) < 80000]
    for it in range(3000):
        raw = rng.choice(srcs)[:rng.choice([20, 64, 300, 5000])]
        s = bytearray(z.reference_compress(raw))
        j = rng.randrange(len(s))
        s[j] = rng.randrange(256) if rng.random() < 0.5 else s[j] ^ (1 << rng.randrange(8))
        _agree(bytes(s))
    if not LIB:
        pytest.skip("liblz4.so.1 is missing: the reference's rejections were checked, not the agreement")


def _kvs(seed, n, big=False):
    rng = random.Random(seed)
    words = [bytes(rng.randrange(32, 127) for _ in range(rng.randrange(3, 24))) for _ in range(30)]
    kvs = []
    for i in range(n):
        if (i // 40) % 3 == 2:
            v = bytes(rng.randrange(256) for _ in range(rng.randrange(1, 160)))          # stretches that stay raw
        elif i % 17 == 5:
            v = bytes([rng.randrange(256)]) * rng.randrange(1, 700)                      # runs: overlapping matches
        else:
            v = b" ".join(rng.choice(words) for _ in range(rng.randrange(0, 16)))
        if big and i % 25 == 12:
            v = (bytes(range(256)) * 700)[:70000 + 997 * i]                              # blocks of several 64 KB fragments
        kvs.append((o.ikey(b"row%06d/c%d" % (i // 2, i % 2), 900 + i), v))
    return kvs


def _blocks(t):
    off, sz = t.block_handles()
    return [int(x) for x in off], [int(x) for x in sz]


@pytest.mark.parametrize("seed,n,bs,big", [(1, 700, 2048, False), (2, 500, 4096, False), (3, 300, 256, False), (4, 120, 2048, True)])
def test_compress_kernel_writes_the_reference_lz4_data_file(seed, n, bs, big):
    """k_lz4_compress + k_snappy_gather over an assembled data file (the oracle's uncompressed table) = the kLZ4Compression
    data file the reference restatement makes of it, byte for byte: same stored form per block (LZ4 or raw by the 12.5 %
    rule), same offsets, same trailers; every stored LZ4 block decodes (liblz4) to the block it replaced."""
    kvs = _kvs(seed, n, big)
    plain = o.Sst.build(kvs, o.TableOptions(block_size=bs))
    off, _ = _blocks(plain)
    data, foff = z.warp_lz4_compress_table(bytes(plain.data), off)
    want, woff, wsz, types = z.reference_lz4_data_file(plain)
    assert foff == woff + [len(want)]
    assert data == want
    assert 4 in types and (0 in types or bs == 256 or big)
    if LIB:
        poff, psz = _blocks(plain)
        for a, b, t, pa_, pb in zip(woff, wsz, types, poff, psz):
            if t == 4:
                n_, body = z.strip_preamble(data[a:a + b])
                assert z.lib_decompress(LIB, body, n_) == bytes(plain.data)[pa_:pa_ + pb]


def test_decode_kernels_rebuild_the_uncompressed_table():
    """k_snappy_sizes + k_snappy_decode on LZ4 blocks: the image of an LZ4 data file is its uncompressed twin's blocks
    (zeroed trailers), from this encoder's streams and from liblz4's (default and HC); the hand-made malformed streams
    are flagged; on mutated streams the kernels agree with the reference decoder (and so never accept what liblz4
    rejects)."""
    kvs = _kvs(7, 400, big=True)
    plain = o.Sst.build(kvs, o.TableOptions(block_size=4096))
    cdata, coff, csz, _ = z.reference_lz4_data_file(plain)
    poff, psz = _blocks(plain)
    pdata = bytes(plain.data)
    want = b"".join(pdata[a:a + b] + bytes(5) for a, b in zip(poff, psz))
    img, ooff = z.warp_uncompress_blocks(cdata, coff, csz, psz)
    assert img == want and ooff == poff + [len(pdata)]
    raws = [pdata[a:a + b] for a, b in zip(poff, psz)]
    for i in range(200):                                                               # runs and short periods: every overlap
        raws.append(bytes(random.Random(i).randrange(256) for _ in range(i % 40 + 1)) * (i * 37 % 3000 + 1))
    raws.append(bytes(300000))                                                         # 255-byte extension runs of ~1200 bytes
    if LIB:
        modes = [("default", 1), ("fast", 4)] + ([("hc", 9)] if hasattr(LIB, "LZ4_compress_HC") else [])
        for mode, accel in modes:
            blob, offs, sizes = b"", [], []
            for k, r in enumerate(raws):
                c = z.varint(len(r)) + z.lib_compress(LIB, r, mode, accel)
                offs.append(len(blob)); sizes.append(len(c))
                blob += c + bytes([5 if mode == "hc" and k % 2 else 4]) + bytes(4)
            img, _ = z.warp_uncompress_blocks(blob, offs, sizes, [len(r) for r in raws])
            assert img == b"".join(r + bytes(5) for r in raws), mode
    # the malformed set: every hand-made stream is flagged (DEV_ERR_BAD_BLOCK), the control decodes
    for s, what in _hand_made():
        try:
            got, _ = z.warp_uncompress_blocks(s + b"\x04" + bytes(4), [0], [len(s)], [z.strip_preamble(s)[0] if s else 0])
        except RuntimeError as e:
            assert e.args[0] == 3 and not what.endswith("ok?"), what
        else:
            assert what.endswith("ok?") and got[:-5] == b"x" * 20 + b"y" * 6, what
    # mutations: the kernels flag exactly what the reference decoder rejects, and decode the rest to the same bytes
    rng = random.Random(3)
    for it in range(300):
        raw = raws[rng.randrange(len(raws) - 1)][:rng.choice([30, 200, 3000])]
        s = bytearray(z.reference_compress(raw))
        j = rng.randrange(len(s))
        s[j] ^= 1 << rng.randrange(8)
        s = bytes(s)
        exp = _agree(s)
        n = z.strip_preamble(s)[0] if not all(b & 128 for b in s) else 0
        if n >= 1 << 20:
            continue
        try:
            got, _ = z.warp_uncompress_blocks(s + b"\x04" + bytes(4), [0], [len(s)], [n])
        except RuntimeError:
            got = None
        assert (got[:-5] if got is not None else None) == exp, (it, s)


def test_decode_kernels_mixed_codecs_in_one_pass():
    """Raw, Snappy, LZ4 and LZ4HC-labelled blocks side by side in one block list: one sizes pass, one decode launch."""
    kvs = _kvs(11, 500)
    plain = o.Sst.build(kvs, o.TableOptions(block_size=2048))
    poff, psz = _blocks(plain)
    pdata = bytes(plain.data)
    raws = [pdata[a:a + b] for a, b in zip(poff, psz)]
    blob, offs, sizes = b"", [], []
    for k, r in enumerate(raws):
        kind = k % 4
        c = r if kind == 0 else (o.snappy_compress(r) if kind == 1 else z.reference_compress(r))
        offs.append(len(blob)); sizes.append(len(c))
        blob += c + bytes([[0, 1, 4, 5][kind]]) + bytes(4)
    img, _ = z.warp_uncompress_blocks(blob, offs, sizes, [len(r) for r in raws])
    assert img == b"".join(r + bytes(5) for r in raws)


def _compressible_kvs(seed, n, vmax=200):
    rng = random.Random(seed)
    words = [bytes(rng.randrange(32, 127) for _ in range(rng.randrange(3, 24))) for _ in range(40)]
    kvs = []
    for i in range(n):
        if (i // 500) % 4 == 3:
            v = bytes(rng.randrange(256) for _ in range(rng.randrange(1, vmax)))
        else:
            v = b" ".join(rng.choice(words) for _ in range(rng.randrange(0, vmax // 10)))
        kvs.append((o.ikey(b"user%08d/col%d" % (i // 3, i % 3), 500 + i), v))
    return kvs


@pytest.mark.parametrize("enc,filt,bs", [(1, 0, 4096), (2, 1, 2048), (1, 1, 32768)])
def test_host_table_builder_lz4_output(pkg, enc, filt, bs):
    """ybgpu_table_builder with compression 4: the data file equals the reference restatement's LZ4 data file of the
    oracle's uncompressed twin, byte for byte (host_lz4_table); index blocks and the filter index are stored compressed
    too; the host meta reader finds the same handles and separators, and the last-key helper and verify_blocks read it."""
    kvs = _compressible_kvs(31 + enc, 6000)
    topt = dict(block_size=bs, index_block_size=1024, min_keys_per_index_block=8, key_encoding=enc, filter_policy=filt, filter_block_size=4096)
    t = z.host_lz4_table(pkg, kvs, **topt)
    plain = o.Sst.build(kvs, o.TableOptions(**topt))
    _, woff, wsz, types = z.reference_lz4_data_file(plain)
    assert len(t.data) < len(plain.data) * 0.8 and set(types) == {0, 4}
    assert t.block_handles(pkg) == (woff, wsz)
    assert len(t.meta) < len(plain.meta)                                                # index blocks were stored compressed
    assert pkg.sst_separators(t.meta_view()) == pkg.sst_separators(plain.meta_view())
    assert pkg.sst_last_key(t.meta_view(), t.data_view()) == kvs[-1][0]
    assert pkg.sst_verify_blocks(t.meta_view(), t.data_view()) == (len(woff), 0)
    sp = pkg.plan_subcompactions([(t.meta_view(), t.data_view())], 4)
    assert 1 <= len(sp) <= 3 and sp == sorted(sp)


def test_host_decoder_rejects_what_the_reference_rejects(pkg):
    """The host reader's LZ4 decoder (last-key helper, metadata blocks): an LZ4 last data block whose stream is malformed
    under a valid checksum is refused, never read. Mutations of the last block, kept only where the reference decoder
    rejects them; the untouched table reads; LZ4HC labels read the same way."""
    kvs = _compressible_kvs(41, 3000)
    kw = dict(block_size=1024, index_block_size=700, min_keys_per_index_block=4)
    for cut in range(0, 80):
        t = z.host_lz4_table(pkg, kvs[:len(kvs) - cut], **kw)
        toff, tsz = t.block_handles(pkg)
        a, b = toff[-1], tsz[-1]
        if t.data[a + b] == 4:
            break
    else:
        raise AssertionError("no variant with an LZ4 last block")
    last = kvs[len(kvs) - cut - 1][0]
    assert pkg.sst_last_key(t.meta_view(), t.data_view()) == last
    d = bytearray(t.data)
    d[a + b:a + b + 5] = z._trailer(bytes(d[a:a + b]), 5)
    assert pkg.sst_last_key(t.meta_view(), z.np_u8(bytes(d))) == last
    rng = random.Random(8)
    rejected = 0
    for _ in range(300):
        s = bytearray(t.data[a:a + b])
        s[rng.randrange(len(s))] ^= 1 << rng.randrange(8)
        try:
            z.reference_uncompress(bytes(s))
            continue
        except ValueError:
            rejected += 1
        d = bytearray(t.data)
        d[a:a + b + 5] = bytes(s) + z._trailer(bytes(s), 4)
        with pytest.raises(pkg.YbGpuError):
            pkg.sst_last_key(t.meta_view(), z.np_u8(bytes(d)))
    assert rejected > 50


def test_sst_check_supported_routing_precheck_lz4(pkg):
    """Routing by job type before any upload: raw, Snappy, LZ4 and LZ4HC tables of either key encoding are taken
    (counts[1], counts[4], counts[5]); blocks labelled zlib,
    bzip2, xpress or ZSTD are NotSupported with their count; a handle outside the data file or an unreadable metadata file
    is Corruption."""
    cfg = o.GenConfig(seed=23, num_rows=3000, cols=2, versions=2, num_files=1, value_len=40)
    kvs = o.Sst.generate(cfg, 0, o.TableOptions(block_size=2048)).read_all()
    plain = o.Sst.build(kvs, o.TableOptions(block_size=2048))
    lz = z.host_lz4_table(pkg, kvs, block_size=2048)
    nb = len(plain.block_handles()[0])
    assert pkg.sst_check_supported(plain.meta_view(), plain.data_view()) == ("OK", [nb, 0, 0, 0, 0, 0, 0, 0])
    st, counts = pkg.sst_check_supported(lz.meta_view(), lz.data_view())
    assert st == "OK" and counts[4] > 0 and counts[0] + counts[4] == nb and sum(counts) == nb
    snap = o.Sst.build(kvs, o.TableOptions(block_size=2048, compression=1))
    st, counts = pkg.sst_check_supported(snap.meta_view(), snap.data_view())
    assert st == "OK" and counts[1] > 0 and counts[0] + counts[1] == nb and sum(counts[2:]) == 0
    tsp = z.host_lz4_table(pkg, kvs, block_size=2048, key_encoding=2)
    assert pkg.sst_check_supported(tsp.meta_view(), tsp.data_view())[0] == "OK"
    if LIB and hasattr(LIB, "LZ4_compress_HC"):
        meta, data, n = z.library_table(pkg, kvs, LIB, "hc", 5, block_size=2048)
        assert n > 0
        st, counts = pkg.sst_check_supported(np.frombuffer(meta, np.uint8), np.frombuffer(data, np.uint8))
        assert st == "OK" and counts[5] == n and sum(counts) == nb
        assert pkg.sst_verify_blocks(np.frombuffer(meta, np.uint8), np.frombuffer(data, np.uint8)) == (nb, 0)
    off, sz = plain.block_handles()
    for ctype in (2, 3, 6, 7):                                        # kZlib, kBZip2, kXpress, kZSTD (options.h:92-101)
        d = bytearray(plain.data)
        for b in (3, 5):
            d[int(off[b]) + int(sz[b])] = ctype
        st, counts = pkg.sst_check_supported(plain.meta_view(), bytes(d))
        assert st == "NotSupported" and counts[ctype] == 2 and counts[0] == nb - 2
    d = bytearray(plain.data)
    d[int(off[1]) + int(sz[1])] = 9
    assert pkg.sst_check_supported(plain.meta_view(), bytes(d))[0] == "Corruption"
    assert pkg.sst_check_supported(plain.meta_view(), bytes(plain.data)[:int(off[-1]) + 3])[0] == "Corruption"
    assert pkg.sst_check_supported(bytes(plain.meta)[:-7], plain.data_view())[0] == "Corruption"


def test_verify_blocks_lz4(pkg):
    """sst_verify_blocks checks LZ4 blocks like any other: all good, then one flipped bit inside an LZ4 block is bad."""
    kvs = _compressible_kvs(51, 4000)
    t = z.host_lz4_table(pkg, kvs, block_size=2048)
    off, sz = t.block_handles(pkg)
    d = t.data
    assert pkg.sst_verify_blocks(t.meta_view(), t.data_view()) == (len(off), 0)
    j = next(i for i, (a, b) in enumerate(zip(off, sz)) if d[a + b] == 4)
    bad = bytearray(d)
    bad[off[j] + sz[j] // 2] ^= 0x20
    assert pkg.sst_verify_blocks(t.meta_view(), np.frombuffer(bytes(bad), np.uint8)) == (len(off), 1)


def test_unsupported_output_compression_is_refused_before_the_device(pkg):
    """output_compression other than none, Snappy or LZ4 is NotSupported at creation, on the host: the table builder, a
    job, a pipelined compaction (no GPU is needed to get the answer)."""
    for c in (2, 3, 5, 7):
        with pytest.raises(pkg.YbGpuError) as e:
            pkg.HostTableBuilder(compression=c)
        assert e.value.status_name == "NotSupported"
        with pytest.raises(pkg.YbGpuError) as e:
            pkg.GpuCompactionJob(output_compression=c)
        assert e.value.status_name == "NotSupported" and "output_compression" in str(e.value)
    t = o.Sst.build(_compressible_kvs(61, 200), o.TableOptions(block_size=1024))
    with pytest.raises(pkg.YbGpuError) as e:
        pkg.compact_files([(t.meta_view(), t.data_view())], output_compression=2)
    assert e.value.status_name == "NotSupported"
    with pytest.raises(pkg.YbGpuError) as e:
        pkg.compact_files_one_table([(t.meta_view(), t.data_view())], output_compression=5)
    assert e.value.status_name == "NotSupported"
