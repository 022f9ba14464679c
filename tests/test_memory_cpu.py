"""Host pieces of device memory budgets, without a device: the uncompressed image a job will need, read from the
varint32 preambles of raw, Snappy and LZ4 tables, and the planner that cuts a key range in two at a row boundary."""
import importlib

import pytest

import lz4_util as z
import oracle_py as o
from test_gpu_parity import _phrase_runs


@pytest.fixture(scope="module")
def pkg():
    return importlib.import_module("yugabyte-db_b200")


def _expected_image(pkg, sst):
    """Every block's uncompressed contents + 5-byte trailer, from the oracle's reader of each block."""
    meta, data = sst.meta_view(), sst.data_view()
    off, sz, _ = pkg.sst_block_handles(meta)
    total, compressed = 0, 0
    for a, b in zip(off, sz):
        a, b = int(a), int(b)
        t = int(data[a + b])
        if t == 0:
            total += b + 5
            continue
        compressed += 1
        n, shift, p = 0, 0, a
        while True:
            n |= (int(data[p]) & 127) << shift
            shift += 7
            if not data[p] & 128:
                break
            p += 1
        total += n + 5
    return total, compressed


def test_uncompressed_image_of_raw_snappy_and_lz4_tables(pkg):
    runs = _phrase_runs(41, 2, 500)
    raw = o.Sst.build(runs[0], o.TableOptions(block_size=4096))
    snappy = o.Sst.build(runs[0], o.TableOptions(block_size=4096, compression=1))
    lz4 = z.host_lz4_table(pkg, runs[0], block_size=4096)
    img_raw, nc_raw = pkg.sst_uncompressed_bytes(raw.meta_view(), raw.data_view())
    assert nc_raw == 0
    off, sz, _ = pkg.sst_block_handles(raw.meta_view())
    assert img_raw == int(sz.sum()) + 5 * len(sz)
    for t in (snappy, lz4):
        img, nc = pkg.sst_uncompressed_bytes(t.meta_view(), t.data_view())
        assert (img, nc) == _expected_image(pkg, t)
        assert nc > 0
        assert img == img_raw                        # the same blocks, uncompressed: the raw table's bytes


@pytest.mark.parametrize("docdb", [True, False])
def test_split_range_cuts_on_row_boundaries_and_tiles_the_range(pkg, docdb):
    cfg = o.GenConfig(seed=3, num_rows=3000, cols=3, versions=2, num_files=3, value_len=64)
    ssts = o.Sst.generate_all(cfg, o.TableOptions(block_size=2048))
    views = [(s.meta_view(), s.data_view()) for s in ssts]
    user_keys = sorted({k[:-8] for s in ssts for k, _ in s.read_all()})
    row = (lambda uk: uk[:32]) if docdb else (lambda uk: uk)     # the generator's DocKey is 32 bytes
    # cut recursively down to a handful of ranges: every cut lies strictly inside its range, on a row boundary, and the
    # leaves tile the key space in order
    ranges, leaves = [(b"", b"")], []
    while ranges:
        lo, hi = ranges.pop()
        n_in = sum(1 for uk in user_keys if uk >= lo and (not hi or uk < hi))
        if n_in < 600:
            leaves.append((lo, hi))
            continue
        mid = pkg.split_range(views, lo, hi, docdb_keys=docdb)
        assert mid is not None
        assert lo < mid and (not hi or mid < hi)
        ranges += [(mid, hi), (lo, mid)]
    leaves.sort(key=lambda r: r[0])
    assert leaves[0][0] == b"" and leaves[-1][1] == b""
    assert all(a[1] == b[0] for a, b in zip(leaves, leaves[1:]))
    assert len(leaves) > 2
    groups = {}
    for uk in user_keys:
        i = max(j for j, (lo, _) in enumerate(leaves) if uk >= lo)
        groups.setdefault(row(uk), set()).add(i)
    assert all(len(v) == 1 for v in groups.values())          # every row in exactly one range


def test_split_range_stops_at_an_unsplittable_row(pkg):
    """A range that holds one DocKey row (however many blocks its versions fill) has no boundary to cut at."""
    import workloads as w
    runs = [r for r in w.giant_row_runs(3, n_runs=2, small_rows=0) if r]
    ssts = [o.Sst.build(r, o.TableOptions(block_size=1024)) for r in runs]
    views = [(s.meta_view(), s.data_view()) for s in ssts]
    n_entries = sum(len(r) for r in runs)
    # cut until nothing is left to cut: the recursion ends, and the leaves that cannot be cut include the giant row's
    ranges, leaves = [(b"", b"")], []
    while ranges:
        lo, hi = ranges.pop()
        mid = pkg.split_range(views, lo, hi)
        if mid is None:
            leaves.append((lo, hi))
            continue
        assert lo < mid and (not hi or mid < hi)
        ranges += [(mid, hi), (lo, mid)]
        assert len(leaves) + len(ranges) < n_entries
    leaves.sort(key=lambda r: r[0])
    assert all(a[1] == b[0] for a, b in zip(leaves, leaves[1:]))

    def count(lo, hi):
        return sum(1 for r in runs for k, _ in r if k[:-8] >= lo and (not hi or k[:-8] < hi))
    assert max(count(lo, hi) for lo, hi in leaves) >= 1000       # one row of thousands of entries, and no cut inside it
