"""The scale cases shared by tests/test_gpu_scale.py (GPU against the oracle) and tests/test_scale_cpu.py (the oracle alone).

Many passes of the engine are hierarchical, and their upper levels only run past a size threshold: a chunk level, then a
one-CTA scan over the chunk sums that loops once there are more than 1 024 chunks; chain segments, then groups of
segments, then a serial walk over the groups. Each case below is sized to sit on one side of such a threshold, and
`levels()` computes, from the result of the compaction, the quantity that decides it. `assert_crossed()` then checks
every entry of the case's `want`, so a case that drifts off its threshold (a generator change, a new block format)
fails instead of passing without reaching the code it names.

Inputs come from the oracle's generator (`o.GenConfig`): row r has one 32-byte DocKey, `cols` columns and `versions`
versions per column, spread over `files` files. With versions = 1 in a major compaction every entry survives, so the
survivor count is rows x cols exactly. The generator's internal keys are 54 bytes: record stride S = 64.

| threshold (kernel constant) | level computed by levels() | cases |
|---|---|---|
| chain groups of SEG x GROUP_SEGS = 262 144 survivors (`k_group_exit`, `k_chain_groups`) | groups | chain_262143 / _262144 / _262145, chain_850001_dev0, chain_850001_ri1 |
| `k_chain_groups`' straddle branch: the first block start of group g at offset >= SEG, reached by a block of > SEG entries | straddles | straddle_1mb, straddle_256kb |
| P / block-start / filter-key scans, SCAN_CHUNK = 4 096: pc > 1 024 | pc | scan_4194304, scan_4194305 |
| emit scan, EMIT_CHUNK = 2 048: > 1 024 chunks of input entries | emit_chunks | emit_2097152, emit_2097160 |
| QQ, QROWS = 128 rows of ri entries per chunk: > 1 024 chunks | qq_chunks | chain_850001_ri1, scan_4194305 |
| block offsets (`k_u64_chunk_sums`), raw and compressed (`d_foff`): > 1 024 chunks of 4 096 blocks | bc | blocks_4194305_raw, blocks_4194305_snappy (bc = 1 025), blocks_lz4 (bc > 1) |
| filter blocks: exactly max_keys, one more, 3 x max_keys + 1 distinct keys | nfb | filter_max_keys, filter_max_keys_plus_1, filter_3max_keys_plus_1 |
| `k_filter_build_smem` with parts = 1 and a grid-stride loop: nfb > 4 x resident CTAs | filter_parts, filter_grid_stride | filter_128b_grid_stride |
| global-atomics `k_filter_build`: filter block > FILTER_SMEM_MAX = 96 KB | filter_route | filter_128kb, filter_256kb |
| partition in chunks of TILE_CHUNK = 2 048 buckets of H records | buckets | partition_8_files, partition_64_files, partition_general_decode |
| `k_scan_blk_counts`: > 1 024 blocks in one input file | max_file_blocks | partition_8_files, partition_general_decode |
| `k_ingest` tickets: more input blocks than one round of 2 CTAs x SMs x 8 blocks | ticket_rounds | partition_8_files, partition_64_files |

The LZ4 output case stays at bc > 1 (more than 4 096 blocks, not 4 194 304): the LZ4 data file it is compared with is
built by the Python restatement of the encoder (tests/lz4_util.py), block by block.
"""
import functools
import math
from dataclasses import dataclass, field

import oracle_py as o

# kernel constants (yugabyte-db_b200/csrc)
SEG = 4096                     # encode_kernels.cuh: entries per chain segment
GROUP_SEGS = 64                # encode_kernels.cuh: segments per chain group
GROUP = SEG * GROUP_SEGS
SCAN_CHUNK = 4096              # encode_kernels.cuh: P, block starts, filter-key ordinals, block offsets
EMIT_CHUNK = 2048              # engine.cu: k_emit_sums / k_scan_sums
QROWS = 128                    # encode_kernels.cuh: k_qq_sums rows per chunk
CTA_SCAN = 1024                # one-CTA scans (k_scan_u64_single, scan_u32_cta, k_scan_sums) loop past this many chunks
TILE_CHUNK = 2048              # engine.cu: k_bucket_counts / k_build_tiles buckets per CTA
FILTER_SMEM_MAX = 96 * 1024    # encode_kernels.cuh: larger filter blocks take the global-atomics k_filter_build
INGEST_CTAS_PER_SM = 2         # ingest_kernels.cuh: persistent k_ingest CTAs per SM
TICKET_BLOCKS = 8              # ingest_kernels.cuh: blocks claimed per ticket
H100_SMS = 132                 # H100 SXM; the GPU test reads the device's own count


def tile_cap(S):
    """Merge-tile capacity per record stride (DESIGN.md section 4): 74 368 / (S + 41), rounded down to 16."""
    return min(4096, 74368 // (S + 41)) & ~15


def tile_h(S):
    """Target tile size H = 65 % of the capacity (engine.cu, partition): n_buckets = N / H + 2."""
    return tile_cap(S) * 65 // 100


@functools.lru_cache(maxsize=None)
def filter_geometry(filter_block_size):
    """(max_keys, filter block bytes) of the oracle's FixedSizeFilterBits for a filter block of this many bytes."""
    import ctypes as C
    L = o.lib()
    L.orc_fixed_size_filter.restype = C.c_uint64
    L.orc_fixed_size_filter.argtypes = [C.c_uint64, C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint64, C.POINTER(C.c_uint64)]
    params = (C.c_uint64 * 3)()
    out = C.create_string_buffer(filter_block_size + 1024)
    n = L.orc_fixed_size_filter(filter_block_size * 8, b"", 0, out, len(out), params)
    return int(params[0]), int(n)


def max_keys(filter_block_size=65536):
    return filter_geometry(filter_block_size)[0]


@dataclass
class Case:
    id: str
    rows: object                    # int, or a function of max_keys(filter_block_size) for the filter cases
    want: dict                      # level -> exact value, or (op, value) with op in "<", "<=", ">", ">="
    cols: int = 1
    versions: int = 1
    files: int = 8
    value_len: int = 4
    in_block: int = 4096
    in_encoding: int = 1
    block_size: int = 4096
    restart: int = 16
    deviation: int = 10
    filter_block_size: int = 0      # 0: no filter policy
    compression: int = 0            # 0 raw, 1 Snappy, 4 LZ4
    cutoff_version: int = None      # history cutoff just above this version's hybrid time (None: HT_MIN)
    route: str = None               # "fused" / "general": PATH_FUSED_INGEST / PATH_GENERAL_DECODE expected
    seed: int = 5
    tags: tuple = field(default=())

    def num_rows(self):
        return self.rows(max_keys(self.filter_block_size or 65536)) if callable(self.rows) else self.rows

    def gen_config(self):
        return o.GenConfig(seed=self.seed, num_rows=self.num_rows(), cols=self.cols, versions=self.versions,
                           num_files=self.files, value_len=self.value_len)

    def input_options(self):
        return o.TableOptions(block_size=self.in_block, key_encoding=self.in_encoding)

    def output_options(self, compression=None):
        return o.TableOptions(block_size=self.block_size, restart=self.restart, deviation=self.deviation,
                              filter_policy=1 if self.filter_block_size else 0,
                              filter_block_size=self.filter_block_size or 65536,
                              compression=self.compression if compression is None else compression)

    def params(self, cfg):
        cutoff = o.HT_MIN if self.cutoff_version is None else o.ht_from_micros(cfg.base_micros + self.cutoff_version * 1000 + 500)
        return dict(cutoff_ht=cutoff)

    def job_kwargs(self, cfg):
        kw = dict(block_size=self.block_size, restart_interval=self.restart, deviation=self.deviation,
                  output_compression=self.compression, **self.params(cfg))
        if self.filter_block_size:
            kw.update(filter_policy=1, filter_block_size=self.filter_block_size)
        return kw


CASES = [
    # 1. chain groups
    Case("chain_262143", 262143, {"survivors": GROUP - 1, "groups": 1}),
    Case("chain_262144", 262144, {"survivors": GROUP, "groups": 1}),
    Case("chain_262145", 262145, {"survivors": GROUP + 1, "groups": 2}),
    Case("chain_850001_dev0", 850001, {"survivors": 850001, "groups": 4}, deviation=0),
    Case("chain_850001_ri1", 850001, {"survivors": 850001, "groups": 4, "qq_chunks": (">", CTA_SCAN)}, restart=1),
    # 2. blocks longer than a segment across group boundaries (tiny values: about 20 000 / 5 000 entries per block)
    Case("straddle_1mb", 1400000, {"groups": (">=", 5), "longest_block": (">", SEG), "straddles": (">=", 1)},
         value_len=1, block_size=1 << 20),
    Case("straddle_256kb", 1400000, {"groups": (">=", 5), "longest_block": (">", SEG), "straddles": (">=", 1)},
         value_len=1, block_size=1 << 18),
    # 3. long scans: survivors and distinct filter keys at 1 024 / 1 025 chunks of SCAN_CHUNK
    Case("scan_4194304", 4194304, {"survivors": 4194304, "pc": CTA_SCAN, "filter_keys": 4194304, "emit_chunks": (">", CTA_SCAN)},
         value_len=2, filter_block_size=65536),
    Case("scan_4194305", 4194305, {"survivors": 4194305, "pc": CTA_SCAN + 1, "filter_keys": 4194305, "emit_chunks": (">", CTA_SCAN),
                                   "qq_chunks": (">", CTA_SCAN)},
         value_len=2, filter_block_size=65536),
    #    emit scan over input entries, MVCC-heavy: 8 versions per key, the cutoff keeps only the newest
    Case("emit_2097152", 262144, {"input_entries": 2097152, "emit_chunks": CTA_SCAN, "survivors": 262144},
         versions=8, cutoff_version=7),
    Case("emit_2097160", 262145, {"input_entries": 2097160, "emit_chunks": CTA_SCAN + 1, "survivors": 262145},
         versions=8, cutoff_version=7),
    # 4. every entry its own block
    Case("blocks_4194305_raw", 4194305, {"out_blocks": 4194305, "bc": CTA_SCAN + 1}, value_len=2, block_size=1),
    Case("blocks_4194305_snappy", 4194305, {"out_blocks": 4194305, "bc": CTA_SCAN + 1}, value_len=2, block_size=1, compression=1),
    Case("blocks_lz4", 9000, {"out_blocks": 9000, "bc": 3}, value_len=40, block_size=1, compression=4),
    # 5. filter blocks
    #    (two columns per row: every filter key is met twice, the second time it is not new)
    Case("filter_max_keys", lambda mk: mk, {"nfb": 1, "last_filter_block_full": True}, cols=2, filter_block_size=65536),
    Case("filter_max_keys_plus_1", lambda mk: mk + 1, {"nfb": 2, "last_filter_block_keys": 1}, cols=2, filter_block_size=65536),
    Case("filter_3max_keys_plus_1", lambda mk: 3 * mk + 1, {"nfb": 4, "last_filter_block_keys": 1}, filter_block_size=65536),
    Case("filter_128b_grid_stride", 200000, {"filter_route": "smem", "filter_parts": 1, "filter_grid_stride": True},
         filter_block_size=128),
    Case("filter_128kb", lambda mk: 2 * mk + 7, {"nfb": 3, "filter_route": "global"}, filter_block_size=128 * 1024),
    Case("filter_256kb", lambda mk: 2 * mk + 7, {"nfb": 3, "filter_route": "global"}, filter_block_size=256 * 1024),
    # 6. partition and ingest at width: 1.6 M entries
    Case("partition_8_files", 800000, {"buckets": (">", TILE_CHUNK), "max_file_blocks": (">", CTA_SCAN), "ticket_rounds": (">", 1)},
         cols=2, route="fused"),
    Case("partition_64_files", 800000, {"buckets": (">", TILE_CHUNK), "ticket_rounds": (">", 1)}, cols=2, files=64, route="fused"),
    Case("partition_general_decode", 800000, {"buckets": (">", TILE_CHUNK), "max_file_blocks": (">", CTA_SCAN)},
         cols=2, in_encoding=2, route="general"),
]

BY_ID = {c.id: c for c in CASES}


def run_oracle(case, collect_kv=False):
    """Generate the case's inputs and compact them with the oracle. The oracle writes no LZ4, so an LZ4 case's oracle
    table is its uncompressed twin. Returns (GenConfig, input tables, Result, output table or None)."""
    cfg = case.gen_config()
    inputs = o.Sst.generate_all(cfg, case.input_options())
    topt = case.output_options(compression=0 if case.compression == 4 else None)
    mode = o.BUILD_SST | (o.COLLECT_KV if collect_kv else 0)
    exp = o.compact(inputs, o.CompactionParams(**case.params(cfg)), topt, mode=mode)
    return cfg, inputs, exp, exp.sst()


# ---- the oracle's output tables, parsed -----------------------------------------------------------------------------

def _varint(b, p):
    r = s = 0
    while True:
        c = b[p]
        p += 1
        r |= (c & 0x7f) << s
        s += 7
        if c < 0x80:
            return r, p


def _stored_block(data, off, size):
    blk = bytes(data[off:off + size])
    t = data[off + size]
    if t == 1:
        return o.snappy_uncompress(blk)
    assert t == 0, "compressed block type %d" % t
    return blk


def _last_interval(blk, ri, key_encoding=1):
    """(entries in the block, last internal key) from the block's last restart interval: one shared-prefix walk of at
    most ri entries (restart points store their key whole)."""
    nres = int.from_bytes(blk[-4:], "little")
    ro = len(blk) - 4 - 4 * nres
    p = int.from_bytes(blk[ro + 4 * (nres - 1):ro + 4 * nres], "little")
    n, k = 0, b""
    while p < ro:
        sh, p = _varint(blk, p)
        ns, p = _varint(blk, p)
        vl, p = _varint(blk, p)
        k = k[:sh] + blk[p:p + ns]
        p += ns + vl
        n += 1
    assert key_encoding == 1 and n <= ri
    return (nres - 1) * ri + n, k


def block_entry_counts(sst, ri):
    """Entries per data block of a shared-prefix table written with restart interval ri."""
    offs, sizes = sst.block_handles()
    d = sst.data_view()
    return [_last_interval(_stored_block(d, int(a), int(b)), ri)[0] for a, b in zip(offs, sizes)]


def first_last_keys(sst, ri):
    """The table's first and last internal keys (FileMetaData::smallest / largest), read from its first and last blocks."""
    offs, sizes = sst.block_handles()
    d = sst.data_view()
    first = _stored_block(d, int(offs[0]), int(sizes[0]))
    _, p = _varint(first, 0)
    ns, p = _varint(first, p)
    _, p = _varint(first, p)
    last = _stored_block(d, int(offs[-1]), int(sizes[-1]))
    return first[p:p + ns], _last_interval(last, ri)[1]


# ---- levels and thresholds ------------------------------------------------------------------------------------------

def straddles(counts):
    """Group boundaries g at which k_chain_groups takes its straddle branch: the first block start inside group g lies at
    an offset >= SEG, so the block before it (which started in an earlier group) holds more than SEG entries."""
    starts = [0]
    for c in counts[:-1]:
        starts.append(starts[-1] + c)
    n = sum(counts)
    hits = []
    for g in range(1, math.ceil(n / GROUP)):
        first = next((s for s in starts if s >= g * GROUP), None)
        if first is not None and first < min(n, (g + 1) * GROUP) and first - g * GROUP >= SEG:
            hits.append(g)
    return hits


def levels(case, inputs, exp, out_sst, sms=H100_SMS):
    """Every level the case table names, from the inputs and the oracle's result. inputs: the generated tables;
    exp: the oracle's Result; out_sst: its output table (None when nothing survives)."""
    n = int(exp.stats.num_output_records)
    N = int(exp.stats.num_input_records)
    props = out_sst.properties() if out_sst is not None else {}
    nblocks = len(out_sst.block_handles()[0]) if out_sst is not None else 0
    file_blocks = [len(s.block_handles()[0]) for s in inputs]
    L = dict(survivors=n, input_entries=N, out_blocks=nblocks,
             groups=math.ceil(n / GROUP), pc=math.ceil(n / SCAN_CHUNK), emit_chunks=math.ceil(N / EMIT_CHUNK),
             qq_chunks=math.ceil(math.ceil(n / case.restart) / QROWS), bc=math.ceil(nblocks / SCAN_CHUNK),
             buckets=N // tile_h(64) + 2, max_file_blocks=max(file_blocks),
             ticket_rounds=math.ceil(sum(file_blocks) / (INGEST_CTAS_PER_SM * sms * TICKET_BLOCKS)))
    if props:
        assert nblocks == o.varint(props["rocksdb.num.data.blocks"]) and n == o.varint(props["rocksdb.num.entries"])
    if case.block_size >= 1 << 18:
        counts = block_entry_counts(out_sst, case.restart)
        assert sum(counts) == n
        L.update(longest_block=max(counts), straddles=len(straddles(counts)))
    if case.filter_block_size:
        mk, fbytes = filter_geometry(case.filter_block_size)
        nfb = o.varint(props["rocksdb.num.filter.blocks"])
        assert nfb == len(out_sst.filter_blocks())
        # one filter key per row (its DocKey): the generator gives every row a distinct DocKey
        n_keys = case.num_rows()
        assert nfb == max(1, math.ceil(n_keys / mk)), (nfb, n_keys, mk)
        stride = (fbytes + 7) & ~7
        resident = max(1, min(2, 200 * 1024 // (stride + 1024))) * sms
        parts = max(1, min(8, resident // nfb))
        last = n_keys - (nfb - 1) * mk
        L.update(nfb=nfb, filter_keys=n_keys, last_filter_block_keys=last, last_filter_block_full=last == mk,
                 filter_route="smem" if stride <= FILTER_SMEM_MAX else "global",
                 filter_parts=parts, filter_grid_stride=nfb * parts > resident * 4)
    return L


def assert_crossed(case, L):
    for name, want in case.want.items():
        got = L[name]
        if isinstance(want, tuple):
            op, v = want
            ok = {"<": got < v, "<=": got <= v, ">": got > v, ">=": got >= v}[op]
        else:
            ok = got == want
        assert ok, "%s: %s = %r, wants %r" % (case.id, name, got, want)
