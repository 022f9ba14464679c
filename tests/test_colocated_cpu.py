"""Slot 0 of cotable / colocated rows rebuilt from the runs (dev_logic.cuh replay_table_seed, what a merge tile does for
the table it starts in), on the CPU through tests/host_harness/colocated_seed.cc: every row of every such table takes its
table-level overwrite from the input runs cut where the row starts, and the compaction must still equal the oracle's.
Tables have up to a few hundred tombstone versions spread over up to 8 runs."""
import collections
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_py as o
import workloads as w
from test_gpu_colocated import many_tables_runs, many_versions_runs, mixed_runs

_HARNESS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_harness")
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        src = os.path.join(_HARNESS, "colocated_seed.cc")
        so = os.path.join(_HARNESS, "libcolocatedseed.so")
        deps = [src, os.path.join(_HARNESS, "..", "..", "yugabyte-db_b200", "csrc", "dev_logic.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            tmp = so + ".tmp%d" % os.getpid()
            subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-x", "c++", "-shared", "-o", tmp, src], stderr=subprocess.DEVNULL)
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u64 = C.c_void_p, C.c_uint64
        L.cs_compact.argtypes = [C.c_int, vp, vp, vp, vp, vp, C.c_int, u64, C.c_int64, C.c_int, u64, C.c_int, u64,
                                 C.c_char_p, u64, C.c_char_p, u64, C.c_char_p, u64, u64]
        for f in ("cs_keys", "cs_vals", "cs_koff", "cs_voff"):
            getattr(L, f).restype = vp
        L.cs_num.restype = u64
        _LIB = L
    return _LIB


def compact_seeded_from_runs(runs, params):
    """The merged-order device logic with every cotable row seeded from the runs; the kv list, as oracle_py.compact_runs."""
    L = _lib()
    flat = [kv for r in runs for kv in r]
    starts = np.zeros(len(runs) + 1, np.uint64)
    starts[1:] = np.cumsum([len(r) for r in runs])
    kb, ko = o._flat([k for k, _ in flat])
    vb, vo = o._flat([v for _, v in flat])
    luk = params._luk
    if luk is None:
        lasts = [r[-1][0][:-8] for r in runs if r]
        luk = max(lasts) if lasts else b""
    rc = L.cs_compact(len(runs), starts.ctypes.data, kb.ctypes.data, ko.ctypes.data, vb.ctypes.data, vo.ctypes.data,
                      params.retention_enabled, params.primary_cutoff_ht, params.table_ttl_ns,
                      params.retain_delete_markers, params.other_min_ht, params.bottommost_level,
                      params.last_sequence, luk, len(luk), params._lo, len(params._lo), params._up, len(params._up),
                      params.cotables_cutoff_ht)
    assert rc == 0, "device logic error %d" % rc
    n = L.cs_num()
    if n == 0:
        return []
    koff = np.ctypeslib.as_array(C.cast(L.cs_koff(), C.POINTER(C.c_uint64)), (n + 1,)).copy()
    voff = np.ctypeslib.as_array(C.cast(L.cs_voff(), C.POINTER(C.c_uint64)), (n + 1,)).copy()
    keys = C.string_at(L.cs_keys(), int(koff[-1]))
    vals = C.string_at(L.cs_vals(), int(voff[-1]))
    return [(keys[int(koff[i]):int(koff[i + 1])], vals[int(voff[i]):int(voff[i + 1])]) for i in range(n)]


def _check(runs, grid):
    for kw in grid:
        p = o.CompactionParams(**kw)
        assert compact_seeded_from_runs(runs, p) == o.compact_runs(runs, p).kv_list(), kw


@pytest.mark.parametrize("seed", range(4))
def test_many_tombstone_versions_from_runs(seed):
    runs = many_versions_runs(seed, n_tables=8, colocated=seed % 2 == 0, n_runs=1 + 2 * seed, rows=(5, 30))
    versions = collections.Counter(k[:n] for r in runs for k, _ in r for n in [17 if k[:1] == b"y" else 5] if k[n] == ord("!"))
    assert min(versions.values()) >= 20
    _check(runs, w.param_grid())


def test_tombstones_in_one_run_from_runs():
    runs = many_versions_runs(9, n_tables=4, colocated=False, n_runs=8, versions=(150, 300), rows=(5, 20), tomb_run=3)
    _check(runs, w.param_grid())


@pytest.mark.parametrize("colocated", [True, False])
def test_many_small_tables_from_runs(colocated):
    _check(many_tables_runs(20 + colocated, n_tables=300, colocated=colocated, n_runs=3), w.param_grid()[::3])


def test_mixed_keys_from_runs():
    _check(mixed_runs(5, n_runs=3), w.param_grid()[::4])
