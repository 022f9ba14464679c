"""TEST-ONLY helpers of the output-check tests: tables from the product's host writer, damaged copies of them re-sealed
with correct trailers, and the check's judgement on the CPU (tests/host_harness/verify_table.cc over dev_logic.cuh)."""
import ctypes as C
import os
import random
import subprocess

import numpy as np

import lz4_util
import oracle_py as o

_HARNESS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_harness")
_LIB = None
KINDS = {0: "ok", 1: "checksum", 2: "compressed_stream", 3: "entry_parse", 4: "key_order", 5: "entry_count", 6: "contents", 7: "key_too_long"}
OK = (0, 0, 0)


def _lib():
    global _LIB
    if _LIB is None:
        src = os.path.join(_HARNESS, "verify_table.cc")
        so = os.path.join(_HARNESS, "libverifytable.so")
        deps = [src, os.path.join(_HARNESS, "..", "..", "yugabyte-db_b200", "csrc", "dev_logic.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            tmp = so + ".tmp%d" % os.getpid()
            subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-x", "c++", "-shared", "-o", tmp, src], stderr=subprocess.DEVNULL)
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.vt_verify.restype = C.c_uint64
        L.vt_verify.argtypes = [C.c_void_p] * 4 + [C.c_uint32, C.c_int, C.c_uint32] + [C.c_void_p] * 6
        _LIB = L
    return _LIB


def rand_kvs(seed, n, klen=(4, 40), vlen=(0, 120), versions=3):
    """n entries in internal-key order: random user keys with shared prefixes, up to `versions` sequence numbers each."""
    rng = random.Random(seed)
    keys = set()
    while len(keys) < max(1, n // 2):
        keys.add(bytes([rng.choice(b"GHS")]) + bytes(rng.randrange(97, 101) for _ in range(rng.randrange(*klen))))
    out = []
    for k in sorted(keys):
        for s in sorted(rng.sample(range(1, 1000), rng.randrange(1, versions + 1)), reverse=True):
            out.append((o.ikey(k, s), bytes(rng.randrange(256) if rng.random() < 0.3 else 120 for _ in range(rng.randrange(*vlen)))))
    return out[:n]


class Table:
    """A split SST as bytes plus its block handles and key encoding."""

    def __init__(self, data, meta, offs, sizes, key_encoding, restart):
        self.data, self.meta, self.offs, self.sizes = bytearray(data), bytes(meta), list(offs), list(sizes)
        self.key_encoding, self.restart = key_encoding, restart

    def copy(self):
        return Table(self.data, self.meta, self.offs, self.sizes, self.key_encoding, self.restart)

    def types(self):
        return [self.data[a + s] for a, s in zip(self.offs, self.sizes)]

    def reseal(self, b):
        """A correct trailer for whatever block b holds now: only the checks behind the checksum can see the damage."""
        a, s = self.offs[b], self.sizes[b]
        crc = o.crc32c(bytes(self.data[a:a + s + 1]))
        masked = (((crc >> 15) | (crc << 17)) + 0xa282ead8) & 0xffffffff
        self.data[a + s + 1:a + s + 5] = masked.to_bytes(4, "little")


def build_table(pkg, kvs, key_encoding=1, restart=16, block_size=4096, compression=0):
    b = pkg.HostTableBuilder(block_size=block_size, restart_interval=restart, key_encoding=key_encoding, compression=compression)
    for k, v in kvs:
        b.add(k, v)
    data, meta = b.finish()
    offs, sizes, enc = pkg.sst_block_handles(np.frombuffer(meta, np.uint8))
    assert enc == key_encoding
    return Table(data, meta, [int(x) for x in offs], [int(x) for x in sizes], key_encoding, restart)


def _image(t):
    """What ReadBlock hands to BlockIter: per block a verdict on the stored bytes (0 / checksum / compressed stream) and
    the uncompressed contents."""
    img, offs, sizes, pre = bytearray(), [], [], []
    for a, s in zip(t.offs, t.sizes):
        stored, typ = bytes(t.data[a:a + s]), t.data[a + s]
        crc = o.crc32c(stored + bytes([typ]))
        masked = (((crc >> 15) | (crc << 17)) + 0xa282ead8) & 0xffffffff
        kind, raw = 0, stored
        if masked != int.from_bytes(t.data[a + s + 1:a + s + 5], "little"):
            kind = 1
        if typ in (1, 4, 5):
            try:
                raw = o.snappy_uncompress(stored) if typ == 1 else lz4_util.reference_uncompress(stored)
            except Exception:
                kind, raw = kind or 2, b""
        offs.append(len(img)); sizes.append(len(raw)); pre.append(kind)
        img += raw
    return bytes(img) + b"\0" * 8, offs, sizes, pre


def cpu_check(t, expect_kvs=None, block_first=None):
    """The check's judgement on table t: (kind, block, entry) of the first failure — OK = (0, 0, 0) — and the entries
    parsed. expect_kvs + block_first: the entries that belong in the table and where its blocks were cut."""
    img, offs, sizes, pre = _image(t)
    nb = len(offs)
    a_off, a_sz, a_pre = np.array(offs, np.uint64), np.array(sizes, np.uint32), np.array(pre, np.uint8)
    a_img = np.frombuffer(img, np.uint8)
    args = [None] * 5
    keep = []
    if expect_kvs is not None:
        kb, ko = o._flat([k for k, _ in expect_kvs])
        vb, vo = o._flat([v for _, v in expect_kvs])
        bf = np.array(block_first, np.uint32)
        keep = [kb, ko, vb, vo, bf]
        args = [bf.ctypes.data, kb.ctypes.data if kb.size else None, ko.ctypes.data, vb.ctypes.data if vb.size else None, vo.ctypes.data]
    n = C.c_uint64()
    f = _lib().vt_verify(a_img.ctypes.data, a_off.ctypes.data, a_sz.ctypes.data, a_pre.ctypes.data, nb, t.key_encoding,
                         t.restart if expect_kvs is not None else 0, *args, C.byref(n))
    del keep
    if f == 2**64 - 1:
        return OK, n.value
    return (f & 15, f >> 32, (f >> 4) & 0x0fffffff), n.value


def block_first(t):
    """First entry of every block of a good table, plus the total (nblocks + 1 numbers)."""
    out = [0]
    for b in range(len(t.offs)):
        one = Table(t.data, t.meta, [t.offs[b]], [t.sizes[b]], t.key_encoding, t.restart)
        res, n = cpu_check(one)
        assert res == OK
        out.append(out[-1] + n)
    return out


def parse_block(raw, key_encoding):
    """Offsets inside an uncompressed shared-prefix block: [(entry start, header length, non_shared, value_len)], the
    restart array's offset and the restart count."""
    assert key_encoding == 1
    nres = int.from_bytes(raw[-4:], "little")
    roff = len(raw) - 4 - 4 * nres
    p, ents = 0, []
    while p < roff:
        q, f = p, []
        for _ in range(3):
            v, sh = 0, 0
            while True:
                c = raw[q]; q += 1
                v |= (c & 127) << sh; sh += 7
                if not c & 128:
                    break
            f.append(v)
        ents.append((p, q - p, f[1], f[2]))
        p = q + f[1] + f[2]
    return ents, roff, nres


def byte_mutations(t, b, seed):
    """Damaged copies of raw (uncompressed, shared-prefix) table t, one flipped bit each inside block b, every one
    re-sealed with a correct trailer: name -> Table."""
    rng = random.Random(seed)
    a, s = t.offs[b], t.sizes[b]
    ents, roff, nres = parse_block(bytes(t.data[a:a + s]), t.key_encoding)
    e = ents[min(len(ents) - 1, max(1, len(ents) // 2))]
    with_val = next((x for x in ents if x[3] > 0), None)
    spots = {"key_delta": e[0] + e[1] + rng.randrange(max(1, e[2])), "shared_varint": e[0], "non_shared_varint": e[0] + 1,
             "value_len_varint": e[0] + e[1] - 1, "restart_count": s - 4 + rng.randrange(2)}
    if nres > 1:
        spots["restart_offset"] = roff + 4 * (nres - 1) + rng.randrange(2)
    if with_val:
        spots["value"] = with_val[0] + with_val[1] + with_val[2] + rng.randrange(with_val[3])
    out = {}
    for name, pos in spots.items():
        m = t.copy()
        m.data[a + pos] ^= 1 << rng.randrange(7)
        m.reseal(b)
        out[name] = m
    return out


def kv_mutations(kvs, bf, b):
    """Entry-level damage at block b of the table cut at bf: name -> the entry list a broken writer would have stored."""
    i = (bf[b] + bf[b + 1]) // 2
    i = min(max(i, 1), len(kvs) - 2)
    out = {"swapped": kvs[:i] + [kvs[i + 1], kvs[i]] + kvs[i + 2:], "duplicated": kvs[:i + 1] + [kvs[i]] + kvs[i + 1:],
           "dropped": kvs[:i] + kvs[i + 1:], "truncated": kvs[:-1]}
    if b + 2 < len(bf):
        out["blocks_swapped"] = kvs[:bf[b]] + kvs[bf[b + 1]:bf[b + 2]] + kvs[bf[b]:bf[b + 1]] + kvs[bf[b + 2]:]
    return out
