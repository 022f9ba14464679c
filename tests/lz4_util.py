"""LZ4 helpers shared by the LZ4 tests:
* the system liblz4 through ctypes and pyarrow's lz4_raw (independent implementations of the format);
* a plain-Python restatement of the engine's LZ4 encoder (host_sst.cc Lz4Compress, lz4_kernels.cuh k_lz4_compress) and
  a strict decoder, the references the engine's writers and readers are compared with;
* the LZ4 kernels' source on emulated warps (tests/host_harness/lz4_emu.cc);
* LZ4 tables: written by the engine's host writer and checked against the restatement, or re-stored from liblz4."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_py as o

_HARNESS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_harness")


def liblz4():
    """liblz4.so.1, or None when the system does not have it."""
    try:
        L = C.CDLL("liblz4.so.1")
    except OSError:
        return None
    for f in ("LZ4_decompress_safe", "LZ4_compress_default", "LZ4_compress_fast", "LZ4_compressBound"):
        if not hasattr(L, f):
            return None
    return L


def pyarrow_lz4():
    try:
        import pyarrow as pa
    except ImportError:
        return None
    return pa if pa.Codec.is_available("lz4_raw") else None


def varint(n):
    out = b""
    while n >= 128:
        out += bytes([(n & 127) | 128])
        n >>= 7
    return out + bytes([n])


def strip_preamble(stream):
    """A stored block (varint32 length + raw LZ4 block) -> (announced length, raw LZ4 block)."""
    n, shift, i = 0, 0, 0
    while True:
        b = stream[i]
        n |= (b & 127) << shift
        i += 1
        if not b & 128:
            return n, stream[i:]
        shift += 7


def lib_decompress(L, body, n):
    """LZ4_decompress_safe with capacity n: the bytes, or None when liblz4 rejects the stream (or returns fewer)."""
    dst = C.create_string_buffer(max(1, n))
    r = L.LZ4_decompress_safe(body, dst, len(body), n)
    return dst.raw[:r] if r >= 0 else None


def lib_compress(L, raw, mode="default", accel=1):
    """A raw LZ4 block from liblz4: LZ4_compress_default, _fast(accel) or _HC(level accel)."""
    cap = L.LZ4_compressBound(len(raw))
    dst = C.create_string_buffer(max(1, cap))
    if mode == "hc":
        n = L.LZ4_compress_HC(raw, dst, len(raw), cap, accel)
    elif mode == "fast":
        n = L.LZ4_compress_fast(raw, dst, len(raw), cap, accel)
    else:
        n = L.LZ4_compress_default(raw, dst, len(raw), cap)
    assert n > 0 or not raw
    return dst.raw[:n]


def parse(body):
    """A raw LZ4 block -> [(literals, match length or 0, offset)]; the format's own parse, no validation."""
    seqs, p = [], 0
    while True:
        tok = body[p]
        p += 1
        lit = tok >> 4
        if lit == 15:
            while True:
                b = body[p]
                p += 1
                lit += b
                if b != 255:
                    break
        lits = body[p:p + lit]
        p += lit
        if p == len(body):
            seqs.append((lits, 0, 0))
            return seqs
        off = body[p] | (body[p + 1] << 8)
        p += 2
        m = tok & 15
        if m == 15:
            while True:
                b = body[p]
                p += 1
                m += b
                if b != 255:
                    break
        seqs.append((lits, m + 4, off))


def _ext(v):
    out = b""
    v -= 15
    while v >= 255:
        out += b"\xff"
        v -= 255
    return out + bytes([v])


def encode(seqs):
    out = bytearray()
    for lits, mlen, off in seqs:
        L, M = len(lits), (mlen - 4 if mlen else 0)
        out.append((min(L, 15) << 4) | min(M, 15))
        if L >= 15:
            out += _ext(L)
        out += lits
        if mlen:
            out += bytes([off & 255, off >> 8])
            if M >= 15:
                out += _ext(M)
    return bytes(out)


def pad_to(body, raw, size):
    """The library's stream grown to exactly `size` bytes by turning match bytes into literals (the last byte of a match
    becomes the first literal of the next sequence), or None when it is longer than that or cannot be grown exactly.
    The parse otherwise stays the library's: its offsets, overlaps and length-extension patterns."""
    if len(body) > size:
        return None
    seqs = [list(s) for s in parse(body)]
    pos = []                                                  # output position where each sequence's match starts
    at = 0
    for lits, mlen, _ in seqs:
        at += len(lits)
        pos.append(at)
        at += mlen
    cur = len(body)
    i = 0
    while cur < size and i < len(seqs) - 1:
        lits, mlen, off = seqs[i]
        if mlen <= 4:
            i += 1
            continue
        nxt = seqs[i + 1]
        trial_i = (lits, mlen - 1, off)
        byte = raw[pos[i] + mlen - 1:pos[i] + mlen]
        trial_n = (byte + nxt[0], nxt[1], nxt[2])
        d = len(encode([trial_i, trial_n])) - len(encode([tuple(seqs[i]), tuple(nxt)]))
        if cur + d > size:
            i += 1
            continue
        seqs[i], seqs[i + 1] = list(trial_i), list(trial_n)
        cur += d
    if cur != size:
        return None
    out = encode([tuple(s) for s in seqs])
    assert len(out) == size
    return out


def _trailer(stored, t):
    c = o.crc32c(stored + bytes([t]))
    return bytes([t]) + (((((c >> 15) | (c << 17)) & 0xffffffff) + 0xa282ead8) & 0xffffffff).to_bytes(4, "little")


def library_table(pkg, kvs, L, mode, stored_type, **topt):
    """(meta, data) of a table whose LZ4 data blocks were re-stored from liblz4's output (mode "default" or "hc") under
    trailer type `stored_type` (4 or 5) with recomputed checksums; the metadata file is the engine writer's LZ4 twin's,
    so every re-stored stream is grown to its slot (pad_to). Also returns how many blocks were re-stored."""
    ours = host_lz4_table(pkg, kvs, **topt)
    plain = o.Sst.build(kvs, o.TableOptions(**_oracle_opts(topt)))
    data = bytearray(ours.data)
    pdata = bytes(plain.data)
    off, sz = ours.block_handles(pkg)
    poff, psz = plain.block_handles()
    n = 0
    for a, b, pa_, pb in zip(off, sz, poff, psz):
        a, b, pa_, pb = int(a), int(b), int(pa_), int(pb)
        if data[a + b] != 4:
            continue
        raw = pdata[pa_:pa_ + pb]
        pre = varint(len(raw))
        body = pad_to(lib_compress(L, raw, mode, 9 if mode == "hc" else 1), raw, b - len(pre))
        if body is None:
            continue
        assert lib_decompress(L, body, len(raw)) == raw
        stored = pre + body
        data[a:a + b + 5] = stored + _trailer(stored, stored_type)
        n += 1
    return bytes(ours.meta), bytes(data), n


def np_u8(b):
    return np.frombuffer(b, np.uint8)


# ---- the reference restatement of the engine's encoder, and a strict decoder -------------------------------------------
def reference_compress(raw):
    """varint32 length + the raw LZ4 block the engine's encoder writes for `raw` (the algorithm of host_sst.cc
    Lz4Compress, statement for statement): 64 KB fragments, 2^12 u16 slots zeroed per fragment, hash
    (w * 0x1e35a7bd) >> 20, greedy with no skipping, positions p <= n - 12 tried, matches ended by min(fragment end, n - 5),
    literal runs spanning fragments, one literals-only sequence at the end."""
    raw = bytes(raw)
    n = len(raw)
    out = bytearray(varint(n))
    lit = 0

    def sequence(to, mlen, off):
        nonlocal lit
        L, M = to - lit, (mlen - 4 if mlen else 0)
        out.append((min(L, 15) << 4) | min(M, 15))
        if L >= 15:
            out.extend(_ext(L))
        out.extend(raw[lit:to])
        if mlen:
            out.extend((off & 255, off >> 8))
            if M >= 15:
                out.extend(_ext(M))

    for fs in range(0, n, 65536):
        m = min(65536, n - fs)
        smax = min(m, n - fs - 8) if n - fs > 8 else 0
        emax = min(m, n - fs - 5) if n - fs > 5 else 0
        table = [0] * 4096
        i = 0
        while i + 4 <= smax:
            w = int.from_bytes(raw[fs + i:fs + i + 4], "little")
            h = ((w * 0x1e35a7bd) & 0xffffffff) >> 20
            cand = table[h]
            table[h] = i
            if cand < i and raw[fs + cand:fs + cand + 4] == raw[fs + i:fs + i + 4]:
                ln = 4
                while i + ln + 64 <= emax and raw[fs + cand + ln:fs + cand + ln + 64] == raw[fs + i + ln:fs + i + ln + 64]:
                    ln += 64
                while i + ln < emax and raw[fs + cand + ln] == raw[fs + i + ln]:
                    ln += 1
                sequence(fs + i, ln, i - cand)
                i += ln
                lit = fs + i
            else:
                i += 1
    sequence(n, 0, 0)
    return bytes(out)


def reference_uncompress(stream):
    """A stored LZ4 block (varint32 length + raw LZ4 block) -> its contents; ValueError on whatever LZ4_decompress_safe
    rejects with the announced length as the capacity (truncations, offset 0 or before the start, a stream ending in a
    match, a match starting within the last 12 bytes or ending within the last 5) and on an output of another length."""
    stream = bytes(stream)
    ulen, shift, p = 0, 0, 0
    while True:
        if p >= len(stream) or p >= 5:
            raise ValueError("bad length preamble")
        b = stream[p]
        ulen |= (b & 127) << shift
        p += 1
        shift += 7
        if not b & 128:
            break
    ulen &= 0xffffffff
    out, e = bytearray(), len(stream)

    def ext(v):
        nonlocal p
        while True:
            if p >= e:
                raise ValueError("truncated length")
            b = stream[p]
            p += 1
            v += b
            if v > ulen:
                raise ValueError("longer than announced")
            if b != 255:
                return v

    while True:
        if p >= e:
            raise ValueError("truncated token")
        tok = stream[p]
        p += 1
        lit = tok >> 4
        if lit == 15:
            lit = ext(lit)
        if e - p < lit or len(out) + lit > ulen:
            raise ValueError("bad literal")
        out += stream[p:p + lit]
        p += lit
        if p == e:
            break
        if len(out) + 12 > ulen or e - p < 2:
            raise ValueError("match position")
        off = stream[p] | (stream[p + 1] << 8)
        p += 2
        ml = tok & 15
        if ml == 15:
            ml = ext(ml)
        ml += 4
        if off == 0 or off > len(out) or len(out) + ml + 5 > ulen:
            raise ValueError("bad match")
        start = len(out) - off
        for k in range(ml):
            out.append(out[start + k])
    if len(out) != ulen:
        raise ValueError("shorter than announced")
    return bytes(out)


def reference_lz4_data_file(plain):
    """The kLZ4Compression data file of an uncompressed table (oracle Sst): each block re-stored as reference_compress
    output when that is shorter than 7/8 of it (GoodCompressionRatio), type 4, checksum over the stored bytes + type.
    Returns (data file, block offsets, block sizes, types)."""
    d = bytes(plain.data)
    out, offs, sizes, types = bytearray(), [], [], []
    for a, b in zip(*plain.block_handles()):
        a, b = int(a), int(b)
        raw = d[a:a + b]
        c = reference_compress(raw)
        stored, t = (c, 4) if len(c) < b - b // 8 else (raw, 0)
        offs.append(len(out)); sizes.append(len(stored)); types.append(t)
        out += stored + _trailer(stored, t)
    return bytes(out), offs, sizes, types


# ---- LZ4 tables --------------------------------------------------------------------------------------------------------
def _oracle_opts(topt):
    m = dict(topt)
    if "restart_interval" in m:
        m["restart"] = m.pop("restart_interval")
    return m


class Table:
    """A split SST held as bytes, with the views the binding and the test helpers take."""

    def __init__(self, meta, data):
        self.meta, self.data = bytes(meta), bytes(data)

    def meta_view(self):
        return np_u8(self.meta)

    def data_view(self):
        return np_u8(self.data)

    def block_handles(self, pkg):
        off, sz, _ = pkg.sst_block_handles(self.meta_view())
        return [int(x) for x in off], [int(x) for x in sz]

    def types(self, pkg):
        return [self.data[a + b] for a, b in zip(*self.block_handles(pkg))]


def host_lz4_table(pkg, kvs, **topt):
    """The table the engine's host writer (ybgpu_table_builder, compression 4) makes of kvs; its data file is checked
    against the reference restatement applied to the oracle's uncompressed twin, byte for byte."""
    b = pkg.HostTableBuilder(compression=4, **topt)
    for k, v in kvs:
        b.add(k, v)
    data, meta = b.finish()
    want, _, _, _ = reference_lz4_data_file(o.Sst.build(kvs, o.TableOptions(**_oracle_opts(topt))))
    assert bytes(data) == want
    return Table(meta, data)


# ---- the LZ4 kernels' source on emulated warps -------------------------------------------------------------------------
_EMU = None


def emu_lib():
    global _EMU
    if _EMU is None:
        src = os.path.join(_HARNESS, "lz4_emu.cc")
        so = os.path.join(_HARNESS, "liblz4emu.so")
        deps = [src, os.path.join(_HARNESS, "warp_emu.cc")] + [
            os.path.join(_HARNESS, "..", "..", "yugabyte-db_b200", "csrc", f) for f in ("snappy_kernels.cuh", "lz4_kernels.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            tmp = so + ".tmp%d" % os.getpid()
            subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-o", tmp, src], stderr=subprocess.DEVNULL)
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.we_lz4_compress_table.restype = C.c_uint64
        L.we_lz4_compress_table.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
        L.we_uncompress_table.restype = C.c_uint64
        L.we_uncompress_table.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p]
        _EMU = L
    return _EMU


def warp_lz4_compress_table(data_file, offsets):
    """k_lz4_compress + k_snappy_gather over an uncompressed data file (blocks + trailers back to back; offsets = the
    blocks' start offsets): (LZ4 data file, final block offsets incl. the end)."""
    raw = np.frombuffer(data_file, np.uint8)
    off = np.array(list(offsets) + [len(data_file)], np.uint64)
    out = np.zeros(len(data_file) + 64, np.uint8)
    foff = np.zeros(len(off), np.uint64)
    n = emu_lib().we_lz4_compress_table(raw.ctypes.data, off.ctypes.data, len(off) - 1, out.ctypes.data, foff.ctypes.data)
    return out[:n].tobytes(), [int(x) for x in foff]


def warp_uncompress_blocks(data_file, offsets, sizes, usizes):
    """k_snappy_sizes + k_snappy_decode over blocks of any codec mix (the output sized from the known contents sizes):
    (uncompressed image, its block offsets incl. the end); RuntimeError(device error code) when the kernels flag a block."""
    raw = np.frombuffer(data_file, np.uint8)
    off = np.array(list(offsets), np.uint64)
    sz = np.array(list(sizes), np.uint32)
    cap = 64 + sum(int(u) + 5 for u in usizes)
    out = np.zeros(cap, np.uint8)
    ooff = np.zeros(len(off) + 1, np.uint64)
    n = emu_lib().we_uncompress_table(raw.ctypes.data, raw.size, off.ctypes.data, sz.ctypes.data, len(off), out.ctypes.data, cap, ooff.ctypes.data)
    if n > 2**63:
        raise RuntimeError(2**64 - 1 - n)
    return out[:n].tobytes(), [int(x) for x in ooff]
