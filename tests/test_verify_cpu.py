"""The output check's judgement, proven without a GPU: dev_logic.cuh's verify_interval and the joins k_verify_blocks makes
between intervals and blocks run on the CPU (tests/host_harness/verify_table.cc) over tables from the product's host
writer — good ones in both key encodings, raw / Snappy / LZ4, and damaged ones re-sealed with correct trailers so that
only the checks behind the checksum can catch them. Plus the ABI of the new entry points."""
import ctypes as C
import importlib
import os
import re

import numpy as np
import pytest

import verify_util as vu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def pkg():
    import __graft_entry__ as g
    g.build()
    return importlib.import_module("yugabyte-db_b200")


@pytest.mark.parametrize("compression", [0, 1, 4])
@pytest.mark.parametrize("restart", [1, 4, 16])
@pytest.mark.parametrize("key_encoding", [1, 2])
def test_good_tables_pass(pkg, key_encoding, restart, compression):
    for seed, block_size in enumerate([256, 4096, 65536]):
        kvs = vu.rand_kvs(100 * key_encoding + 10 * restart + seed, 900)
        t = vu.build_table(pkg, kvs, key_encoding, restart, block_size, compression)
        bf = vu.block_first(t)
        assert bf[-1] == len(kvs)
        assert vu.cpu_check(t) == (vu.OK, len(kvs))
        assert vu.cpu_check(t, kvs, bf) == (vu.OK, len(kvs))
        if compression and block_size >= 4096:
            assert any(x == compression for x in t.types())


def test_single_entry_and_many_restart_rounds(pkg):
    t = vu.build_table(pkg, vu.rand_kvs(3, 1), restart=16)
    assert vu.cpu_check(t, vu.rand_kvs(3, 1), [0, 1]) == (vu.OK, 1)
    kvs = vu.rand_kvs(4, 700, vlen=(0, 8))
    t = vu.build_table(pkg, kvs, restart=1, block_size=65536)       # hundreds of intervals per block: many rounds of 32
    assert len(t.offs) == 1
    assert vu.cpu_check(t, kvs, [0, 700]) == (vu.OK, 700)


# what each kind of damage may be reported as, with and without the entries that belong in the table
_BYTE_KINDS = {
    "key_delta": ({"key_order", "contents"}, {"key_order", "ok"}),
    "value": ({"contents"}, {"ok"}),
    "shared_varint": ({"entry_parse", "key_order", "contents"}, {"entry_parse", "key_order", "ok"}),
    "non_shared_varint": ({"entry_parse", "key_order", "contents"}, {"entry_parse", "key_order", "ok"}),
    "value_len_varint": ({"entry_parse", "key_order", "contents"}, {"entry_parse", "key_order", "ok"}),
    "restart_offset": ({"entry_parse", "key_order", "contents", "entry_count"}, {"entry_parse", "key_order", "ok"}),
    "restart_count": ({"entry_parse", "key_order", "contents", "entry_count"}, {"entry_parse", "key_order", "ok"}),
}


@pytest.mark.parametrize("restart", [1, 4, 16])
def test_flipped_bits_behind_a_correct_trailer(pkg, restart):
    kvs = vu.rand_kvs(40 + restart, 1200)
    t = vu.build_table(pkg, kvs, 1, restart, 2048)
    bf = vu.block_first(t)
    assert len(t.offs) > 6
    seen = set()
    for b in (0, len(t.offs) // 2, len(t.offs) - 1):
        for seed in range(6):
            for name, m in vu.byte_mutations(t, b, 1000 * b + seed).items():
                (kind, blk, ent), _ = vu.cpu_check(m, kvs, bf)
                assert vu.KINDS[kind] in _BYTE_KINDS[name][0], (name, b, seed, vu.KINDS[kind])
                assert blk == b, (name, b, seed, blk)
                assert bf[b] + ent < bf[b + 1] or vu.KINDS[kind] == "entry_count"
                (kind2, blk2, _), _ = vu.cpu_check(m)
                assert vu.KINDS[kind2] in _BYTE_KINDS[name][1], (name, b, seed, vu.KINDS[kind2])
                assert kind2 == 0 or blk2 in (b, b + 1)
                seen.add(vu.KINDS[kind])
    assert {"entry_parse", "key_order", "contents"} <= seen


def test_flipped_bit_without_resealing_is_a_checksum_failure(pkg):
    kvs = vu.rand_kvs(7, 600)
    for compression in (0, 1, 4):
        t = vu.build_table(pkg, kvs, 1, 16, 2048, compression)
        b = len(t.offs) // 2
        m = t.copy()
        m.data[t.offs[b] + t.sizes[b] // 2] ^= 0x10
        assert vu.cpu_check(m)[0] == (1, b, 0)
        if compression:
            assert t.types()[b] == compression
            m.reseal(b)                       # the damaged stream behind a correct trailer
            (kind, blk, _), _ = vu.cpu_check(m, kvs, vu.block_first(t))
            if vu._image(m)[0] == vu._image(t)[0]:
                assert kind == 0              # e.g. another copy offset inside a run of equal bytes: the same contents
            else:
                assert kind != 0 and blk == b


@pytest.mark.parametrize("key_encoding", [1, 2])
@pytest.mark.parametrize("compression", [0, 1])
def test_entry_level_damage(pkg, key_encoding, compression):
    kvs = vu.rand_kvs(90 + key_encoding, 1500)
    good = vu.build_table(pkg, kvs, key_encoding, 16, 2048, compression)
    bf = vu.block_first(good)
    b = len(bf) // 2
    # against the entries that belong there the first wrong entry is reported, before the order breaks behind it
    want = {"swapped": {"contents"}, "duplicated": {"key_order"}, "dropped": {"contents", "entry_count"},
            "truncated": {"entry_count"}, "blocks_swapped": {"contents"}}
    for name, bad_kvs in vu.kv_mutations(kvs, bf, b).items():
        m = vu.build_table(pkg, bad_kvs, key_encoding, 16, 2048, compression)
        (kind, blk, ent), _ = vu.cpu_check(m, kvs, bf)
        assert vu.KINDS[kind] in want[name], (name, vu.KINDS[kind])
        # everything before the damage is the good table's bytes, so the report names the block the damage starts in
        assert blk == (len(bf) - 2 if name == "truncated" else b), (name, blk, b)
        (kind2, blk2, _), _ = vu.cpu_check(m)                 # the table alone: a shorter table is still a table
        assert vu.KINDS[kind2] == ("ok" if name in ("dropped", "truncated") else "key_order"), (name, vu.KINDS[kind2])
        assert kind2 == 0 or blk2 in (b, b + 1), (name, blk2, b)


def test_abi_of_the_check(pkg):
    L = pkg.lib()
    hdr = open(os.path.join(ROOT, "include", "ybgpu_compaction.h")).read()
    body = hdr.split("typedef struct ybgpu_output_check {")[1].split("}")[0]
    fields = re.findall(r"\b(uint64_t|uint32_t|double)\s+(\w+);", body)
    ctype = {"uint64_t": C.c_uint64, "uint32_t": C.c_uint32, "double": C.c_double}
    assert [(n, ctype[t]) for t, n in fields] == list(pkg.OutputCheck._fields_)
    assert C.sizeof(pkg.OutputCheck) == 56
    kinds = dict((n.lower(), int(v)) for n, v in re.findall(r"YBGPU_CHECK_([A-Z_]+)\s*=\s*(\d+)", hdr))
    assert kinds == {v: k for k, v in pkg.CHECK_KIND_NAMES.items()} == {v: k for k, v in vu.KINDS.items()}
    assert int(re.search(r"YBGPU_PATH_OUTPUT_VERIFIED = (\d+)", hdr).group(1)) == pkg.PATH_OUTPUT_VERIFIED == 8192
    L.ybgpu_job_verify_output.argtypes = [C.c_void_p, C.c_void_p]
    chk = pkg.OutputCheck()
    assert L.ybgpu_job_verify_output(None, C.byref(chk)) == 4
    L.ybgpu_sst_verify_device.argtypes = [C.c_int32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p]
    assert L.ybgpu_sst_verify_device(0, None, 0, None, 0, C.byref(chk)) == 4
    t = vu.build_table(pkg, vu.rand_kvs(1, 50))
    meta = np.frombuffer(t.meta, np.uint8)
    assert L.ybgpu_sst_verify_device(0, meta.ctypes.data, meta.size, None, 10, C.byref(chk)) == 4
    assert L.ybgpu_sst_verify_device(0, meta.ctypes.data, meta.size, meta.ctypes.data, meta.size, None) == 4
    junk = np.zeros(64, np.uint8)
    assert L.ybgpu_sst_verify_device(0, junk.ctypes.data, junk.size, junk.ctypes.data, junk.size, C.byref(chk)) == 2   # no footer: before any device is touched
    for name in ("ybgpu_compact_files_checked", "ybgpu_compact_files_one_table_checked"):
        assert hasattr(L, name)
