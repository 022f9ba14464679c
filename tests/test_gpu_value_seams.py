"""The block assembler's value copy at every seam, against the oracle byte for byte: k_encode_v5 moves a value as
destination-aligned 16-byte chunks with the bytes in front of the first / behind the last whole chunk stored one by one.

Values of 1-101 bytes and of 4 KB-70 KB are placed at every one of the 32 destination residues (checked on the oracle's
table before the GPU runs), so every seam case occurs: no whole chunk, exactly one, no edge bytes and the longest edges,
source and destination misaligned either way. TTL-carrying values under a table TTL are rewritten by the compaction (a
new prefix, the rest copied from behind the old one), and tombstones carry no value bytes to copy."""
import importlib
import random

import numpy as np
import pytest

import dockv_util as dk
import oracle_py as o
import workloads as w
from test_gpu_parity import check, runs_to_ssts
from test_gpu_routes import has

pytestmark = pytest.mark.gpu

SHORT = list(range(1, 102))
LONG = [4096, 4097, 4127, 4128, 4129, 8191, 16384 + 17, 32768 - 5, 65536 + 3, 70 * 1024]


@pytest.fixture(scope="module")
def pkg():
    m = importlib.import_module("yugabyte-db_b200")
    assert m.device_count() >= 1, "GPU tests need a CUDA device"
    return m


def _varint(b, p):
    v = s = 0
    while True:
        c = b[p]; p += 1
        v |= (c & 0x7f) << s; s += 7
        if c < 0x80:
            return v, p


def value_residues(data, meta, pkg):
    """{value length: set of file offsets mod 32 of the values' first byte} over every entry of a shared-prefix table."""
    offs, sizes, enc = pkg.sst_block_handles(np.frombuffer(meta, dtype=np.uint8))
    assert enc == 1
    out = {}
    for off, size in zip(offs, sizes):
        off, size = int(off), int(size)
        blk = data[off:off + size]
        nres = int.from_bytes(blk[-4:], "little")
        end = size - 4 - 4 * nres
        p = 0
        while p < end:
            _, p = _varint(blk, p)
            nk, p = _varint(blk, p)
            vl, p = _varint(blk, p)
            p += nk
            out.setdefault(vl, set()).add((off + p) % 32)
            p += vl
    return out


def runs(seed, lengths, per_length, ttl_share=0.0):
    """Two runs of one-column rows; key padding varies the destination offsets."""
    rng = random.Random(seed)
    order = [L for L in lengths for _ in range(per_length)]
    rng.shuffle(order)
    rows = []
    for L in order:
        pad = "p" * rng.randrange(0, 40)
        uk = dk.sub_doc_key(dk.doc_key(["k%06d_%s" % (len(rows), pad)]), [dk.kcol(1)], ht=(w.BASE_US + 10 * rng.randrange(5), 0, 0))
        body = bytes(rng.randrange(256) for _ in range(min(L, 64))) * (L // 64 + 1)
        v = dk.vstr(body[:L - 1]) if L > 1 else dk.TOMBSTONE
        if rng.random() < ttl_share:
            v = dk.with_ttl(v, rng.choice([1, 50, 10**7]))
        rows.append((uk, v))
    out = [[], []]
    for n, (uk, v) in enumerate(rows):
        out[n % 2].append((o.ikey(uk, (1 << 50) + n), v))
    return [w.sort_run(r) for r in out]


def _every_residue(ssts, pkg, lengths, block_size):
    exp = o.compact(ssts, o.CompactionParams(**w.param_grid()[0]), o.TableOptions(block_size=block_size))
    res = value_residues(exp.sst().data, exp.sst().meta, pkg)
    missing = {L: 32 - len(res.get(L, ())) for L in lengths if len(res.get(L, ())) < 32}
    assert not missing, missing


def test_short_values_every_residue(pkg):
    ssts = runs_to_ssts(runs(1, SHORT, 360, ttl_share=0.2), 4096)
    _every_residue(ssts, pkg, [L for L in SHORT if L > 1], 4096)
    for kw in (w.param_grid()[0], w.param_grid()[8], w.param_grid()[9]):
        for enc in (1, 2):
            job, _ = check(pkg, ssts, block_size=4096, output_key_encoding=enc, **kw)
            assert has(job.stats(), pkg.PATH_ENCODER_V5)


def test_long_values_every_residue(pkg):
    ssts = runs_to_ssts(runs(7, LONG, 200, ttl_share=0.2), 16384)
    _every_residue(ssts, pkg, LONG, 32768)
    for kw in (w.param_grid()[0], w.param_grid()[8]):
        for bs in (4096, 32768):
            job, _ = check(pkg, ssts, block_size=bs, **kw)
            assert has(job.stats(), pkg.PATH_ENCODER_V5)


def test_verify_output_after_the_split(pkg):
    ssts = runs_to_ssts(runs(3, SHORT[::7] + LONG[::3], 24, ttl_share=0.2), 8192)
    job, _ = check(pkg, ssts, block_size=8192, filter_policy=1, **w.param_grid()[8])
    chk = job.verify_output()
    assert chk.failure_kind == 0 and has(job.stats(), pkg.PATH_OUTPUT_VERIFIED)
    assert chk.entries_parsed == job.stats().num_output_records
