"""ctypes binding of libybgpu.so (include/ybgpu_compaction.h)."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libybgpu.so")

HT_MIN = 0
HT_MAX = 2**64 - 1
HT_INVALID = 2**64 - 2
TTL_MAX_NS = 2**63 - 1
MAX_SEQUENCE = (1 << 56) - 1

STATUS_NAMES = {0: "OK", 1: "NotFound", 2: "Corruption", 3: "NotSupported", 4: "InvalidArgument", 5: "IOError",
                7: "RuntimeError", 9: "IllegalState", 25: "TryAgain", 27: "ShutdownInProgress"}


class YbGpuError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__("%s: %s" % (STATUS_NAMES.get(status, status), msg))
        self.status = status
        self.status_name = STATUS_NAMES.get(status, str(status))


class JobOptions(C.Structure):
    _fields_ = [
        ("device", C.c_int32), ("bottommost_level", C.c_int32), ("last_sequence", C.c_uint64),
        ("largest_user_key", C.c_char_p), ("largest_user_key_len", C.c_uint64), ("has_largest_user_key", C.c_int32),
        ("retention_enabled", C.c_int32), ("history_cutoff_ht", C.c_uint64), ("cotables_cutoff_ht", C.c_uint64),
        ("table_ttl_ns", C.c_int64), ("retain_delete_markers_in_major_compaction", C.c_int32),
        ("other_min_ht", C.c_uint64),
        ("key_bounds_lower", C.c_char_p), ("key_bounds_lower_len", C.c_uint64),
        ("key_bounds_upper", C.c_char_p), ("key_bounds_upper_len", C.c_uint64),
        ("block_size", C.c_uint32), ("block_restart_interval", C.c_int32), ("block_size_deviation", C.c_int32),
        ("output_key_encoding", C.c_int32), ("index_block_size", C.c_uint32), ("min_keys_per_index_block", C.c_uint32),
        ("verify_checksums", C.c_int32),
        ("range_lower", C.c_char_p), ("range_lower_len", C.c_uint64),
        ("range_upper", C.c_char_p), ("range_upper_len", C.c_uint64),
        ("cuda_stream", C.c_void_p),
        ("filter_policy", C.c_int32), ("filter_block_size", C.c_uint32),
        ("yield_fn", C.c_void_p), ("yield_ctx", C.c_void_p),
        ("compute_user_boundary_values", C.c_int32),
        ("output_compression", C.c_int32),
        ("device_memory_budget", C.c_uint64),
    ]


YIELD_FN = C.CFUNCTYPE(None, C.c_void_p)


class UserValue(C.Structure):
    _fields_ = [("tag", C.c_uint32), ("len", C.c_uint32), ("value", C.c_uint8 * 256)]


class BlockHandle(C.Structure):
    _fields_ = [("offset", C.c_uint64), ("size", C.c_uint64)]


class JobStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "num_input_records", "num_output_records", "num_record_drop_hidden", "num_record_drop_obsolete",
        "num_record_drop_feed", "total_input_raw_key_bytes", "total_input_raw_value_bytes",
        "total_output_raw_key_bytes", "total_output_raw_value_bytes", "num_output_data_blocks",
        "output_data_file_size", "output_meta_file_size", "smallest_seqno", "largest_seqno")] + [
        ("gpu_seconds", C.c_double), ("gpu_kernel_launches", C.c_uint32), ("h2d_bytes", C.c_uint64),
        ("d2h_bytes", C.c_uint64), ("phase_seconds", C.c_double * 8), ("phase_launches", C.c_uint32 * 8),
                ("path_flags", C.c_uint32), ("tiles_inside_rows", C.c_uint32), ("device_bytes_peak", C.c_uint64)]

    def as_dict(self):
        d = {n: getattr(self, n) for n, _ in self._fields_}
        d["phase_seconds"] = list(self.phase_seconds)
        d["phase_launches"] = list(self.phase_launches)
        return d


PHASE_NAMES = ["block_scan", "decode", "partition", "merge_filter", "encode"]
PATH_FUSED_INGEST, PATH_GENERAL_DECODE, PATH_SNAPPY, PATH_PARTITION_RETRY, PATH_ENCODER_V4, PATH_ENCODER_V5, PATH_KV_INPUT = 1, 2, 4, 8, 16, 32, 64
PATH_SNAPPY_OUTPUT = 128
PATH_LZ4, PATH_LZ4_OUTPUT = 256, 512
PATH_INGEST_RETRY, PATH_FAST_DECODE, PATH_ENCODER_FUSED = 1024, 2048, 4096
PATH_OUTPUT_VERIFIED = 8192
COMPRESSION_NONE, COMPRESSION_SNAPPY, COMPRESSION_LZ4 = 0, 1, 4   # output_compression (rocksdb::CompressionType)


CHECK_KIND_NAMES = {0: "ok", 1: "checksum", 2: "compressed_stream", 3: "entry_parse", 4: "key_order", 5: "entry_count",
                    6: "contents", 7: "key_too_long"}


class OutputCheck(C.Structure):
    """ybgpu_output_check: what the device-side table check read and, if it failed, where."""
    _fields_ = [("blocks_checked", C.c_uint64), ("blocks_compressed", C.c_uint64), ("entries_parsed", C.c_uint64),
                ("bytes_read", C.c_uint64), ("gpu_seconds", C.c_double), ("failure_kind", C.c_uint32),
                ("failure_block", C.c_uint32), ("failure_entry", C.c_uint32), ("reserved", C.c_uint32)]

    @property
    def failure(self):
        return CHECK_KIND_NAMES.get(self.failure_kind, str(self.failure_kind))


class OutputCheckError(YbGpuError):
    """A failed table check: .check is the OutputCheck with the first failure."""

    def __init__(self, status, msg, check):
        super().__init__(status, msg)
        self.check = check


class GenConfig(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("num_rows", C.c_uint64), ("cols", C.c_uint32), ("versions", C.c_uint32),
                ("num_files", C.c_uint32), ("value_len", C.c_uint32), ("base_micros", C.c_uint64),
                ("tombstone_per_1024", C.c_uint32), ("tombstone_newest", C.c_uint32), ("row_offset", C.c_uint64),
                ("hash_rows_total", C.c_uint64)]

    def __init__(self, seed=1, num_rows=1000, cols=1, versions=1, num_files=2, value_len=256,
                 base_micros=1790000000 * 1000000, tombstone_per_1024=0, tombstone_newest=0, row_offset=0,
                 hash_rows_total=0):
        super().__init__(seed, num_rows, cols, versions, num_files, value_len, base_micros, tombstone_per_1024,
                         tombstone_newest, row_offset, hash_rows_total)


_LIB = None


def lib():
    """Loads libybgpu.so; raises (never falls back) when the CUDA library is not built."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise ImportError("libybgpu.so is not built (run __graft_entry__.build()); "
                          "there is no CPU fallback for the compaction engine")
    L = C.CDLL(LIB_PATH)
    vp, u64 = C.c_void_p, C.c_uint64
    L.ybgpu_job_options_init.argtypes = [C.POINTER(JobOptions)]
    L.ybgpu_job_create.argtypes = [C.POINTER(JobOptions), C.POINTER(vp)]
    L.ybgpu_job_destroy.argtypes = [vp]
    L.ybgpu_job_error.argtypes = [vp]
    L.ybgpu_job_error.restype = C.c_char_p
    L.ybgpu_last_error.restype = C.c_char_p
    L.ybgpu_job_add_input.argtypes = [vp, vp, u64, vp, u64, C.c_int32, u64]
    L.ybgpu_job_add_input_device.argtypes = [vp, vp, u64, vp, u64, C.c_int32, u64]
    L.ybgpu_job_add_input_sst.argtypes = [vp, vp, u64, vp, u64, u64]
    L.ybgpu_job_wait_inputs.argtypes = [vp]
    L.ybgpu_job_set_cotable_filters.argtypes = [vp, vp, vp, C.c_uint32]
    L.ybgpu_job_add_input_kv.argtypes = [vp, vp, vp, vp, vp, u64]
    L.ybgpu_job_run.argtypes = [vp, vp]
    L.ybgpu_job_get_stats.argtypes = [vp, C.POINTER(JobStats)]
    L.ybgpu_job_kv_stream_sizes.argtypes = [vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]
    L.ybgpu_job_fetch_kv_stream.argtypes = [vp, vp, vp, vp, vp]
    L.ybgpu_job_output_sizes.argtypes = [vp, C.POINTER(u64), C.POINTER(u64)]
    L.ybgpu_job_fetch_output.argtypes = [vp, vp, u64, vp, u64]
    L.ybgpu_job_output_boundaries.argtypes = [vp, vp, C.POINTER(u64), vp, C.POINTER(u64)]
    L.ybgpu_job_kv_stream_digest.argtypes = [vp, C.POINTER(u64)]
    L.ybgpu_job_emit_kv_stream.argtypes = [vp, vp, vp]
    L.ybgpu_gen_ssts.argtypes = [C.POINTER(GenConfig), C.POINTER(JobOptions), C.POINTER(vp), C.c_int32]
    L.ybgpu_gen_sst.argtypes = [C.POINTER(GenConfig), C.c_uint32, C.POINTER(JobOptions), C.POINTER(vp)]
    L.ybgpu_sst_free.argtypes = [vp]
    L.ybgpu_sst_data.argtypes = [vp, C.POINTER(u64)]
    L.ybgpu_sst_data.restype = vp
    L.ybgpu_sst_meta.argtypes = [vp, C.POINTER(u64)]
    L.ybgpu_sst_meta.restype = vp
    L.ybgpu_sst_num_entries.argtypes = [vp]
    L.ybgpu_sst_num_entries.restype = u64
    L.ybgpu_sst_raw_bytes.argtypes = [vp]
    L.ybgpu_sst_raw_bytes.restype = u64
    L.ybgpu_device_count.restype = C.c_int32
    L.ybgpu_version.restype = C.c_char_p
    _LIB = L
    return L


def device_count():
    return lib().ybgpu_device_count()


def bind_thread_to_device(device):
    """ybgpu_bind_thread_to_device: CPU affinity + preferred memory node of the calling thread (and of threads it
    creates later) = the NUMA node of `device`. Returns (numa_node, num_cpus); (-1, 0) when nothing was done."""
    node, ncpu = C.c_int32(-1), C.c_int32(0)
    lib().ybgpu_bind_thread_to_device(device, C.byref(node), C.byref(ncpu))
    return node.value, ncpu.value


def _np_ptr(a):
    return a.ctypes.data if a.size else None


EMIT_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64)
STREAM_PRIVATE = 2**64 - 1      # YBGPU_STREAM_PRIVATE: a non-blocking stream owned by the job


def make_options(device=0, bottommost=True, last_sequence=MAX_SEQUENCE, largest_user_key=None,
                 retention=True, cutoff_ht=HT_MIN, cotables_cutoff_ht=HT_INVALID, table_ttl_ns=TTL_MAX_NS,
                 retain_delete_markers=False, other_min_ht=HT_MAX, lower=b"", upper=b"", block_size=32768,
                 restart_interval=16, deviation=10, output_key_encoding=1, index_block_size=32768,
                 min_keys_per_index_block=100, verify_checksums=True, cuda_stream=None, range_lower=b"", range_upper=b"",
                 filter_policy=0, filter_block_size=65536, yield_fn=None, user_boundary_values=False,
                 output_compression=0, device_memory_budget=0):
    """ybgpu_job_options from keyword arguments; returns (options, objects to keep alive). yield_fn: a Python
    callable() invoked at the engine's yield points (PauseIfNecessary). device_memory_budget: bytes of HBM the job
    (or the whole pipelined compaction) may hold at once, 0 = unlimited."""
    L = lib()
    o = JobOptions()
    L.ybgpu_job_options_init(C.byref(o))
    o.device = device
    o.bottommost_level = int(bottommost)
    o.last_sequence = last_sequence
    if largest_user_key is not None:
        o.largest_user_key, o.largest_user_key_len, o.has_largest_user_key = largest_user_key, len(largest_user_key), 1
    o.retention_enabled = int(retention)
    o.history_cutoff_ht = cutoff_ht
    o.cotables_cutoff_ht = cotables_cutoff_ht
    o.table_ttl_ns = table_ttl_ns
    o.retain_delete_markers_in_major_compaction = int(retain_delete_markers)
    o.other_min_ht = other_min_ht
    o.key_bounds_lower, o.key_bounds_lower_len = lower, len(lower)
    o.key_bounds_upper, o.key_bounds_upper_len = upper, len(upper)
    o.block_size, o.block_restart_interval, o.block_size_deviation = block_size, restart_interval, deviation
    o.output_key_encoding = output_key_encoding
    o.index_block_size, o.min_keys_per_index_block = index_block_size, min_keys_per_index_block
    o.verify_checksums = int(verify_checksums)
    o.filter_policy, o.filter_block_size = filter_policy, filter_block_size
    o.cuda_stream = cuda_stream
    o.range_lower, o.range_lower_len = range_lower, len(range_lower)
    o.range_upper, o.range_upper_len = range_upper, len(range_upper)
    o.compute_user_boundary_values = int(bool(user_boundary_values))
    o.output_compression = int(output_compression)
    o.device_memory_budget = int(device_memory_budget)
    cb = None
    if yield_fn is not None:
        cb = YIELD_FN(lambda _ctx: yield_fn())
        o.yield_fn = C.cast(cb, C.c_void_p)
    return o, (largest_user_key, lower, upper, range_lower, range_upper, cb)


class GpuCompactionJob:
    """One rocksdb::CompactionJob::Run on the GPU (compaction_job.cc:521-589)."""

    def __init__(self, device=0, bottommost=True, last_sequence=MAX_SEQUENCE, largest_user_key=None,
                 retention=True, cutoff_ht=HT_MIN, cotables_cutoff_ht=HT_INVALID, table_ttl_ns=TTL_MAX_NS,
                 retain_delete_markers=False, other_min_ht=HT_MAX, lower=b"", upper=b"", block_size=32768,
                 restart_interval=16, deviation=10, output_key_encoding=1, index_block_size=32768,
                 min_keys_per_index_block=100, verify_checksums=True, cuda_stream=None, range_lower=b"", range_upper=b"",
                 filter_policy=0, filter_block_size=65536, yield_fn=None, user_boundary_values=False, output_compression=0,
                 device_memory_budget=0):
        L = lib()
        o, self._keep = make_options(device, bottommost, last_sequence, largest_user_key, retention, cutoff_ht,
                                     cotables_cutoff_ht, table_ttl_ns, retain_delete_markers, other_min_ht, lower, upper,
                                     block_size, restart_interval, deviation, output_key_encoding, index_block_size,
                                     min_keys_per_index_block, verify_checksums, cuda_stream, range_lower, range_upper,
                                     filter_policy, filter_block_size, yield_fn, user_boundary_values, output_compression,
                                     device_memory_budget)
        h = C.c_void_p()
        st = L.ybgpu_job_create(C.byref(o), C.byref(h))
        if st != 0:
            raise YbGpuError(st, L.ybgpu_last_error().decode())
        self.h = h
        self._inputs = []

    def close(self):
        if getattr(self, "h", None):
            lib().ybgpu_job_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, st):
        if st != 0:
            raise YbGpuError(st, lib().ybgpu_job_error(self.h).decode())

    def add_input(self, data, offsets, sizes, key_encoding=1, ht_filter=HT_INVALID):
        """data: numpy uint8 array (host) of the data file; offsets/sizes: block handles."""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        hs = np.zeros((len(offsets), 2), dtype=np.uint64)
        hs[:, 0] = offsets
        hs[:, 1] = sizes
        self._check(lib().ybgpu_job_add_input(self.h, _np_ptr(data), data.size, _np_ptr(hs), len(offsets), key_encoding, ht_filter))

    def add_input_device(self, dev_ptr, length, offsets, sizes, key_encoding=1, ht_filter=HT_INVALID):
        hs = np.zeros((len(offsets), 2), dtype=np.uint64)
        hs[:, 0] = offsets
        hs[:, 1] = sizes
        self._check(lib().ybgpu_job_add_input_device(self.h, dev_ptr, length, _np_ptr(hs), len(offsets), key_encoding, ht_filter))

    def add_input_kv(self, kvs):
        """A sorted run held in memory (the flush path's input): kvs = [(internal key, value)] in internal-key order."""
        keys = np.frombuffer(b"".join(k for k, _ in kvs), dtype=np.uint8) if kvs else np.zeros(0, np.uint8)
        vals = np.frombuffer(b"".join(v for _, v in kvs), dtype=np.uint8) if kvs else np.zeros(0, np.uint8)
        koff = np.zeros(len(kvs) + 1, np.uint64)
        voff = np.zeros(len(kvs) + 1, np.uint64)
        if kvs:
            koff[1:] = np.cumsum([len(k) for k, _ in kvs])
            voff[1:] = np.cumsum([len(v) for _, v in kvs])
        self._inputs.append((keys, vals, koff, voff))
        self._check(lib().ybgpu_job_add_input_kv(self.h, _np_ptr(keys) if keys.size else None, _np_ptr(koff), _np_ptr(vals) if vals.size else None,
                                                 _np_ptr(voff), len(kvs)))

    def set_cotable_filters(self, db_oids, hybrid_times):
        """Per-database cotable HybridTime filters of the input added last (sorted database oids, a hybrid time each)."""
        oids = np.ascontiguousarray(db_oids, dtype=np.uint32)
        hts = np.ascontiguousarray(hybrid_times, dtype=np.uint64)
        assert oids.size == hts.size
        self._check(lib().ybgpu_job_set_cotable_filters(self.h, _np_ptr(oids), _np_ptr(hts), oids.size))

    def wait_inputs(self):
        """Blocks until the queued host->device copies of the inputs have completed."""
        self._check(lib().ybgpu_job_wait_inputs(self.h))

    def add_input_sst(self, meta, data, ht_filter=HT_INVALID):
        meta = np.ascontiguousarray(meta, dtype=np.uint8)
        data = np.ascontiguousarray(data, dtype=np.uint8)
        self._inputs.append((meta, data))
        self._check(lib().ybgpu_job_add_input_sst(self.h, _np_ptr(meta), meta.size, _np_ptr(data), data.size, ht_filter))

    def run(self):
        self._check(lib().ybgpu_job_run(self.h, None))
        return self.stats()

    def stats(self):
        s = JobStats()
        self._check(lib().ybgpu_job_get_stats(self.h, C.byref(s)))
        return s

    def kv_stream_sizes(self):
        n, kb, vb = C.c_uint64(), C.c_uint64(), C.c_uint64()
        self._check(lib().ybgpu_job_kv_stream_sizes(self.h, C.byref(n), C.byref(kb), C.byref(vb)))
        return n.value, kb.value, vb.value

    def fetch_kv_stream(self):
        n, kb, vb = self.kv_stream_sizes()
        keys = np.zeros(kb + 1, np.uint8)
        vals = np.zeros(vb + 1, np.uint8)
        koff = np.zeros(n + 1, np.uint64)
        voff = np.zeros(n + 1, np.uint64)
        self._check(lib().ybgpu_job_fetch_kv_stream(self.h, keys.ctypes.data, koff.ctypes.data, vals.ctypes.data, voff.ctypes.data))
        return keys[:kb], koff, vals[:vb], voff

    def kv_list(self):
        keys, koff, vals, voff = self.fetch_kv_stream()
        kb, vb = keys.tobytes(), vals.tobytes()
        return [(kb[int(koff[i]):int(koff[i + 1])], vb[int(voff[i]):int(voff[i + 1])]) for i in range(len(koff) - 1)]

    def output_sizes(self):
        dl, ml = C.c_uint64(), C.c_uint64()
        self._check(lib().ybgpu_job_output_sizes(self.h, C.byref(dl), C.byref(ml)))
        return dl.value, ml.value

    def fetch_output(self, data_buf=None, meta_buf=None):
        """Copies <n>.sst.sblock.0 and <n>.sst into the given uint8 numpy buffers (allocated here when
        None). Returns views trimmed to the file sizes."""
        if data_buf is not None and meta_buf is not None:
            # caller-provided (pinned) buffers: one call, the metadata file is built on the host while the
            # data file is in flight
            self._check(lib().ybgpu_job_fetch_output(self.h, data_buf.ctypes.data, data_buf.size, meta_buf.ctypes.data, meta_buf.size))
            dl, ml = self.output_sizes()
            return data_buf[:dl], meta_buf[:ml]
        dl, ml = self.output_sizes()
        data = data_buf if data_buf is not None else np.empty(dl + 1, np.uint8)
        meta = meta_buf if meta_buf is not None else np.empty(ml + 1, np.uint8)
        self._check(lib().ybgpu_job_fetch_output(self.h, data.ctypes.data, data.size, meta.ctypes.data, meta.size))
        return data[:dl], meta[:ml]

    def boundaries(self):
        a, b = C.create_string_buffer(4096), C.create_string_buffer(4096)
        al, bl = C.c_uint64(), C.c_uint64()
        self._check(lib().ybgpu_job_output_boundaries(self.h, a, C.byref(al), b, C.byref(bl)))
        return a.raw[:al.value], b.raw[:bl.value]

    def emit_kv_stream(self, fn):
        """ybgpu_job_emit_kv_stream: fn(key: bytes, value: bytes) -> int is called for every surviving entry in
        output order (the CompactionFeed::Feed shape); a non-zero return aborts with that status."""
        def tramp(_ctx, k, kl, v, vl):
            return int(fn(C.string_at(k, kl), C.string_at(v, vl)) or 0)
        cb = EMIT_FN(tramp)
        self._check(lib().ybgpu_job_emit_kv_stream(self.h, C.cast(cb, C.c_void_p), None))

    def user_values(self):
        """ybgpu_job_output_user_values -> (smallest, largest): {tag: encoded key component}."""
        L = lib()
        L.ybgpu_job_output_user_values.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
        a, b = (UserValue * 32)(), (UserValue * 32)()
        n = C.c_uint32()
        self._check(L.ybgpu_job_output_user_values(self.h, a, b, 32, C.byref(n)))
        return ({a[i].tag: bytes(a[i].value[:a[i].len]) for i in range(n.value)},
                {b[i].tag: bytes(b[i].value[:b[i].len]) for i in range(n.value)})

    def verify_output(self):
        """ybgpu_job_verify_output: re-reads the finished table on the GPU (checksums, compressed streams, every entry,
        key order, contents against the merge result). Returns the OutputCheck; raises OutputCheckError on a failure."""
        L = lib()
        L.ybgpu_job_verify_output.argtypes = [C.c_void_p, C.POINTER(OutputCheck)]
        chk = OutputCheck()
        st = L.ybgpu_job_verify_output(self.h, C.byref(chk))
        if st != 0:
            raise OutputCheckError(st, L.ybgpu_job_error(self.h).decode(), chk)
        return chk

    def digest(self):
        d = C.c_uint64()
        self._check(lib().ybgpu_job_kv_stream_digest(self.h, C.byref(d)))
        return d.value


class HostTableBuilder:
    """rocksdb::TableBuilder-shaped host writer (ybgpu_table_builder_*)."""

    def __init__(self, block_size=32768, restart_interval=16, deviation=10, index_block_size=32768,
                 min_keys_per_index_block=100, key_encoding=1, filter_policy=0, filter_block_size=65536, compression=0):
        L = lib()
        L.ybgpu_table_builder_create.argtypes = [C.POINTER(JobOptions), C.POINTER(C.c_void_p)]
        L.ybgpu_table_builder_add.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint64]
        L.ybgpu_table_builder_finish.argtypes = [C.c_void_p]
        L.ybgpu_table_builder_destroy.argtypes = [C.c_void_p]
        L.ybgpu_table_builder_num_entries.argtypes = [C.c_void_p]
        L.ybgpu_table_builder_num_entries.restype = C.c_uint64
        L.ybgpu_table_builder_files.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64),
                                                C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
        o = JobOptions()
        L.ybgpu_job_options_init(C.byref(o))
        o.block_size, o.block_restart_interval, o.block_size_deviation = block_size, restart_interval, deviation
        o.index_block_size, o.min_keys_per_index_block, o.output_key_encoding = index_block_size, min_keys_per_index_block, key_encoding
        o.filter_policy, o.filter_block_size = filter_policy, filter_block_size
        o.output_compression = compression
        self.h = C.c_void_p()
        st = L.ybgpu_table_builder_create(C.byref(o), C.byref(self.h))
        if st != 0:
            raise YbGpuError(st, L.ybgpu_last_error().decode())

    def add(self, key, value):
        st = lib().ybgpu_table_builder_add(self.h, key, len(key), value, len(value))
        if st != 0:
            raise YbGpuError(st, "table builder add")

    def finish(self):
        L = lib()
        st = L.ybgpu_table_builder_finish(self.h)
        if st != 0:
            raise YbGpuError(st, "table builder finish")
        d, m, dl, ml = C.c_void_p(), C.c_void_p(), C.c_uint64(), C.c_uint64()
        L.ybgpu_table_builder_files(self.h, C.byref(d), C.byref(dl), C.byref(m), C.byref(ml))
        return C.string_at(d, dl.value), C.string_at(m, ml.value)

    def __del__(self):
        if getattr(self, "h", None):
            lib().ybgpu_table_builder_destroy(self.h)
            self.h = None


class GeneratedSst:
    """A synthetic split SST made by the product's generator (ybgpu_gen_ssts)."""

    def __init__(self, handle):
        self.h = handle

    def __del__(self):
        if getattr(self, "h", None) and _LIB is not None:
            _LIB.ybgpu_sst_free(self.h)
            self.h = None

    def _view(self, fn):
        n = C.c_uint64()
        p = fn(self.h, C.byref(n))
        if n.value == 0:
            return np.zeros(0, np.uint8)
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), (n.value,))

    def data_view(self):
        return self._view(lib().ybgpu_sst_data)

    def meta_view(self):
        return self._view(lib().ybgpu_sst_meta)

    @property
    def num_entries(self):
        return lib().ybgpu_sst_num_entries(self.h)

    @property
    def raw_bytes(self):
        return lib().ybgpu_sst_raw_bytes(self.h)


def generate_ssts(cfg, block_size=32768, restart_interval=16, max_threads=None):
    L = lib()
    o = JobOptions()
    L.ybgpu_job_options_init(C.byref(o))
    o.block_size, o.block_restart_interval = block_size, restart_interval
    arr = (C.c_void_p * cfg.num_files)()
    st = L.ybgpu_gen_ssts(C.byref(cfg), C.byref(o), arr, max_threads or os.cpu_count() or 1)
    if st != 0:
        raise YbGpuError(st, "synthetic SST generation failed")
    return [GeneratedSst(arr[i]) for i in range(cfg.num_files)]


def generate_sst_files(cfg, file_indices, block_size=32768, restart_interval=16, max_threads=None):
    """Only the files `file_indices` of the synthetic tablet `cfg` (ybgpu_gen_sst per file, on threads): what one rank
    of a key-range sharded compaction holds."""
    import threading
    L = lib()
    o = JobOptions()
    L.ybgpu_job_options_init(C.byref(o))
    o.block_size, o.block_restart_interval = block_size, restart_interval
    out = [None] * len(file_indices)
    errs = []

    def work(slot, f):
        h = C.c_void_p()
        st = L.ybgpu_gen_sst(C.byref(cfg), f, C.byref(o), C.byref(h))
        if st != 0:
            errs.append(st)
        else:
            out[slot] = GeneratedSst(h)
    threads = [threading.Thread(target=work, args=(i, f)) for i, f in enumerate(file_indices)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errs:
        raise YbGpuError(errs[0], "synthetic SST generation failed")
    return out


def sst_block_handles(meta):
    """(offsets, sizes, key_encoding) of the data blocks of a split SST, from its metadata file."""
    L = lib()
    L.ybgpu_sst_meta_handles.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_int32)]
    meta = np.ascontiguousarray(meta, dtype=np.uint8)
    n, enc = C.c_uint64(), C.c_int32()
    if L.ybgpu_sst_meta_handles(meta.ctypes.data, meta.size, None, 0, C.byref(n), C.byref(enc)) != 0:
        raise YbGpuError(2, L.ybgpu_last_error().decode())
    hs = np.zeros((n.value, 2), dtype=np.uint64)
    if n.value and L.ybgpu_sst_meta_handles(meta.ctypes.data, meta.size, hs.ctypes.data, n.value, C.byref(n), C.byref(enc)) != 0:
        raise YbGpuError(2, L.ybgpu_last_error().decode())
    return hs[:, 0].copy(), hs[:, 1].copy(), enc.value


def sst_separators(meta):
    """Index (separator) internal keys of the data blocks, as a list of bytes."""
    L = lib()
    L.ybgpu_sst_meta_separators.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    meta = np.ascontiguousarray(meta, dtype=np.uint8)
    n, nb = C.c_uint64(), C.c_uint64()
    if L.ybgpu_sst_meta_separators(meta.ctypes.data, meta.size, None, 0, None, C.byref(n), C.byref(nb)) != 0:
        raise YbGpuError(2, L.ybgpu_last_error().decode())
    keys = np.zeros(nb.value + 1, np.uint8)
    offs = np.zeros(n.value + 1, np.uint64)
    if L.ybgpu_sst_meta_separators(meta.ctypes.data, meta.size, keys.ctypes.data, keys.size, offs.ctypes.data, C.byref(n), C.byref(nb)) != 0:
        raise YbGpuError(2, L.ybgpu_last_error().decode())
    kb = keys.tobytes()
    return [kb[int(offs[i]):int(offs[i + 1])] for i in range(n.value)]


class InputFile(C.Structure):
    _fields_ = [("meta_file", C.c_void_p), ("meta_file_len", C.c_uint64), ("data_file", C.c_void_p),
                ("data_file_len", C.c_uint64), ("hybrid_time_filter", C.c_uint64),
                ("cotable_db_oids", C.c_void_p), ("cotable_hybrid_times", C.c_void_p), ("num_cotable_filters", C.c_uint64)]


class SubOutput(C.Structure):
    _fields_ = [("data_offset", C.c_uint64), ("data_len", C.c_uint64), ("meta_offset", C.c_uint64), ("meta_len", C.c_uint64),
                ("stats", JobStats), ("range_lower_len", C.c_uint32), ("range_upper_len", C.c_uint32),
                ("range_lower", C.c_uint8 * 256), ("range_upper", C.c_uint8 * 256),
                ("smallest_key_len", C.c_uint32), ("largest_key_len", C.c_uint32),
                ("smallest_key", C.c_uint8 * 1032), ("largest_key", C.c_uint8 * 1032)]

    @property
    def lower(self):
        return bytes(self.range_lower[:self.range_lower_len])

    @property
    def upper(self):
        return bytes(self.range_upper[:self.range_upper_len])

    @property
    def smallest(self):
        return bytes(self.smallest_key[:self.smallest_key_len])

    @property
    def largest(self):
        return bytes(self.largest_key[:self.largest_key_len])


def _input_files(ssts, ht_filters=None, cotable_filters=None):
    """ssts: list of (meta ndarray, data ndarray); cotable_filters: per file None or (sorted database oids, hybrid
    times). Returns (ctypes array, keepalive)."""
    arr = (InputFile * len(ssts))()
    keep = []
    for i, (meta, data) in enumerate(ssts):
        meta = np.ascontiguousarray(meta, dtype=np.uint8)
        data = np.ascontiguousarray(data, dtype=np.uint8)
        keep += [meta, data]
        oid_p, ht_p, ncf = None, None, 0
        if cotable_filters and cotable_filters[i]:
            oids = np.ascontiguousarray(cotable_filters[i][0], dtype=np.uint32)
            hts = np.ascontiguousarray(cotable_filters[i][1], dtype=np.uint64)
            keep += [oids, hts]
            oid_p, ht_p, ncf = oids.ctypes.data, hts.ctypes.data, oids.size
        arr[i] = InputFile(meta.ctypes.data, meta.size, data.ctypes.data, data.size,
                           ht_filters[i] if ht_filters else HT_INVALID, oid_p, ht_p, ncf)
    return arr, keep


def plan_subcompactions(ssts, max_subcompactions, docdb_keys=True):
    """Splitter user keys (row aligned) for at most max_subcompactions key ranges."""
    L = lib()
    L.ybgpu_plan_subcompactions.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32)]
    arr, keep = _input_files(ssts)
    buf = np.zeros((max(1, max_subcompactions), 256), np.uint8)
    lens = np.zeros(max(1, max_subcompactions), np.uint32)
    n = C.c_uint32()
    st = L.ybgpu_plan_subcompactions(arr, len(ssts), max_subcompactions, int(docdb_keys), buf.ctypes.data, lens.ctypes.data, C.byref(n))
    if st != 0:
        raise YbGpuError(st, "plan_subcompactions")
    return [buf[i, :lens[i]].tobytes() for i in range(n.value)]


def split_range(ssts, lower=b"", upper=b"", docdb_keys=True):
    """ybgpu_split_range: the row-aligned splitter halving [lower, upper) of the inputs, or None when no row boundary
    lies inside the range."""
    L = lib()
    L.ybgpu_split_range.argtypes = [C.c_void_p, C.c_uint32, C.c_int32, C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32, C.c_void_p,
                                    C.POINTER(C.c_uint32)]
    arr, keep = _input_files(ssts)
    buf = np.zeros(256, np.uint8)
    n = C.c_uint32()
    st = L.ybgpu_split_range(arr, len(ssts), int(docdb_keys), lower, len(lower), upper, len(upper), buf.ctypes.data, C.byref(n))
    if st == 1:                       # YBGPU_NOT_FOUND
        return None
    if st != 0:
        raise YbGpuError(st, "split_range")
    return buf[:n.value].tobytes()


def sst_uncompressed_bytes(meta, data):
    """ybgpu_sst_uncompressed_bytes: (uncompressed image bytes, blocks stored compressed) of one table, read on the host."""
    L = lib()
    L.ybgpu_sst_uncompressed_bytes.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    meta = np.ascontiguousarray(meta, dtype=np.uint8)
    data = np.ascontiguousarray(data, dtype=np.uint8)
    img, nc = C.c_uint64(), C.c_uint64()
    st = L.ybgpu_sst_uncompressed_bytes(meta.ctypes.data, meta.size, data.ctypes.data, data.size, C.byref(img), C.byref(nc))
    if st != 0:
        raise YbGpuError(st, L.ybgpu_last_error().decode())
    return img.value, nc.value


def sst_last_key(meta, data):
    """Last internal key of a split SST (FileMetaData::largest), read on the host."""
    L = lib()
    L.ybgpu_sst_last_key.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(C.c_uint32)]
    meta = np.ascontiguousarray(meta, dtype=np.uint8)
    data = np.ascontiguousarray(data, dtype=np.uint8)
    out = np.zeros(1032, np.uint8)
    n = C.c_uint32()
    st = L.ybgpu_sst_last_key(meta.ctypes.data, meta.size, data.ctypes.data, data.size, out.ctypes.data, C.byref(n))
    if st != 0:
        raise YbGpuError(st, "sst_last_key")
    return out[:n.value].tobytes()


class SubcompactionResult:
    def __init__(self, outputs, total, data_arena, meta_arena):
        self.outputs, self.total, self.data_arena, self.meta_arena = outputs, total, data_arena, meta_arena

    def files(self):
        """[(data bytes view, meta bytes view)] of the non-empty outputs, in range order."""
        return [(self.data_arena[o.data_offset:o.data_offset + o.data_len], self.meta_arena[o.meta_offset:o.meta_offset + o.meta_len])
                for o in self.outputs if o.data_len]


def compact_files(ssts, max_subcompactions=8, max_in_flight=3, data_arena=None, meta_arena=None, ht_filters=None, cotable_filters=None,
                  verify_outputs=None, output_slots=None, **job_kwargs):
    """ybgpu_compact_files: one compaction as pipelined key-range subcompactions (one output SST per
    range, in range order). ssts: list of (meta ndarray, data ndarray) in host memory. verify_outputs (True / False):
    ybgpu_compact_files_checked, every range's table checked on the GPU before it is copied out. With a
    device_memory_budget, ranges may be cut further: output_slots (default 1024) bounds how many."""
    L = lib()
    L.ybgpu_compact_files.argtypes = [C.POINTER(JobOptions), C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64,
                                      C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(JobStats),
                                      C.c_char_p, C.c_uint64]
    L.ybgpu_compact_files_checked.argtypes = L.ybgpu_compact_files.argtypes + [C.c_int32]
    o, keep_o = make_options(**job_kwargs)
    arr, keep = _input_files(ssts, ht_filters, cotable_filters)
    in_bytes = sum(int(d.size) for _, d in ssts)
    slots = max(1, max_subcompactions) if not o.device_memory_budget else (output_slots or 1024)
    if data_arena is None:
        data_arena = np.empty(in_bytes + (in_bytes >> 4) + (1 << 20) + 4096 * slots, np.uint8)
    if meta_arena is None:
        meta_arena = np.empty((in_bytes >> 5) + (4 << 20) + 4096 * slots, np.uint8)
    outs = (SubOutput * slots)()
    n = C.c_uint32(slots)
    total = JobStats()
    err = C.create_string_buffer(512)
    args = (C.byref(o), arr, len(ssts), max_subcompactions, max_in_flight, data_arena.ctypes.data, data_arena.size,
            meta_arena.ctypes.data, meta_arena.size, None, outs, C.byref(n), C.byref(total), err, 512)
    st = L.ybgpu_compact_files(*args) if verify_outputs is None else L.ybgpu_compact_files_checked(*args, int(bool(verify_outputs)))
    if st != 0:
        raise YbGpuError(st, err.value.decode(errors="replace"))
    return SubcompactionResult([outs[i] for i in range(n.value)], total, data_arena, meta_arena)


class OneTableResult(C.Structure):
    _fields_ = [("data_len", C.c_uint64), ("meta_len", C.c_uint64), ("num_ranges", C.c_uint32), ("num_pieces", C.c_uint32),
                ("smallest_key_len", C.c_uint32), ("largest_key_len", C.c_uint32),
                ("smallest_key", C.c_uint8 * 1032), ("largest_key", C.c_uint8 * 1032)]

    @property
    def smallest(self):
        return bytes(self.smallest_key[:self.smallest_key_len])

    @property
    def largest(self):
        return bytes(self.largest_key[:self.largest_key_len])


def compact_files_one_table(ssts, max_subcompactions=8, max_in_flight=3, data_out=None, meta_out=None, ht_filters=None, cotable_filters=None,
                            verify_outputs=None, **job_kwargs):
    """ybgpu_compact_files_one_table: the pipelined compaction with ONE output table. Returns
    (data view, meta view, OneTableResult, total JobStats). verify_outputs (True / False):
    ybgpu_compact_files_one_table_checked, every range checked on the GPU before it is copied out."""
    L = lib()
    L.ybgpu_compact_files_one_table.argtypes = [C.POINTER(JobOptions), C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64,
                                                C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(OneTableResult), C.POINTER(JobStats),
                                                C.c_char_p, C.c_uint64]
    L.ybgpu_compact_files_one_table_checked.argtypes = L.ybgpu_compact_files_one_table.argtypes + [C.c_int32]
    o, keep_o = make_options(**job_kwargs)
    arr, keep = _input_files(ssts, ht_filters, cotable_filters)
    in_bytes = sum(int(d.size) for _, d in ssts)
    if data_out is None:
        data_out = np.empty(in_bytes + (in_bytes >> 4) + (1 << 20), np.uint8)
    if meta_out is None:
        meta_out = np.empty((in_bytes >> 4) + (4 << 20), np.uint8)
    res = OneTableResult()
    total = JobStats()
    err = C.create_string_buffer(512)
    args = (C.byref(o), arr, len(ssts), max_subcompactions, max_in_flight, data_out.ctypes.data, data_out.size,
            meta_out.ctypes.data, meta_out.size, None, C.byref(res), C.byref(total), err, 512)
    st = L.ybgpu_compact_files_one_table(*args) if verify_outputs is None else L.ybgpu_compact_files_one_table_checked(*args, int(bool(verify_outputs)))
    if st != 0:
        raise YbGpuError(st, err.value.decode(errors="replace"))
    return data_out[:res.data_len], meta_out[:res.meta_len], res, total


class RangeShardResult(C.Structure):
    _fields_ = [("data_len", C.c_uint64), ("meta_len", C.c_uint64), ("num_ranges", C.c_uint32), ("num_pieces", C.c_uint32),
                ("sent_bytes", C.c_uint64), ("received_bytes", C.c_uint64), ("sent_to_peers_bytes", C.c_uint64),
                ("plan_seconds", C.c_double), ("exchange_seconds", C.c_double), ("total_seconds", C.c_double),
                ("range_lower_len", C.c_uint32), ("range_upper_len", C.c_uint32),
                ("range_lower", C.c_uint8 * 256), ("range_upper", C.c_uint8 * 256),
                ("smallest_key_len", C.c_uint32), ("largest_key_len", C.c_uint32),
                ("smallest_key", C.c_uint8 * 1032), ("largest_key", C.c_uint8 * 1032)]

    @property
    def lower(self):
        return bytes(self.range_lower[:self.range_lower_len])

    @property
    def upper(self):
        return bytes(self.range_upper[:self.range_upper_len])

    @property
    def smallest(self):
        return bytes(self.smallest_key[:self.smallest_key_len])

    @property
    def largest(self):
        return bytes(self.largest_key[:self.largest_key_len])


def range_comm_unique_id():
    """ybgpu_range_comm_unique_id: 128 bytes to hand to every rank (one rank creates it)."""
    buf = (C.c_uint8 * 128)()
    st = lib().ybgpu_range_comm_unique_id(buf)
    if st != 0:
        raise YbGpuError(st, "range_comm_unique_id (is libnccl available?)")
    return bytes(buf)


class RangeComm:
    """ybgpu_range_comm: the communicator of a key-range sharded compaction (one process per GPU)."""

    def __init__(self, unique_id, rank, world, device):
        L = lib()
        L.ybgpu_range_comm_create.argtypes = [C.c_char_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]
        L.ybgpu_range_comm_destroy.argtypes = [C.c_void_p]
        h = C.c_void_p()
        st = L.ybgpu_range_comm_create(unique_id, rank, world, device, C.byref(h))
        if st != 0:
            raise YbGpuError(st, "range_comm_create")
        self.h, self.rank, self.world, self.device = h, rank, world, device

    def close(self):
        if getattr(self, "h", None):
            lib().ybgpu_range_comm_destroy(self.h)
            self.h = None

    def compact(self, ssts, rounds=1, chunk_bytes=64 << 20, data_out=None, meta_out=None, ht_filters=None, out_bytes_hint=None, **job_kwargs):
        """ybgpu_compact_range_sharded over this rank's local files [(meta ndarray, data ndarray)]. Returns
        (data view, meta view, RangeShardResult, JobStats) — this rank's table of the sharded compaction."""
        L = lib()
        L.ybgpu_compact_range_sharded.argtypes = [C.c_void_p, C.POINTER(JobOptions), C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint64,
                                                  C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(RangeShardResult),
                                                  C.POINTER(JobStats), C.c_char_p, C.c_uint64]
        job_kwargs.setdefault("device", self.device)
        o, keep_o = make_options(**job_kwargs)
        arr, keep = _input_files(ssts, ht_filters) if ssts else (None, None)
        if data_out is None:
            n = out_bytes_hint if out_bytes_hint is not None else 2 * sum(int(d.size) for _, d in ssts) * self.world + (8 << 20)
            data_out = np.empty(n, np.uint8)
        if meta_out is None:
            meta_out = np.empty((data_out.size >> 4) + (4 << 20), np.uint8)
        res, total = RangeShardResult(), JobStats()
        err = C.create_string_buffer(512)
        st = L.ybgpu_compact_range_sharded(self.h, C.byref(o), arr, len(ssts), rounds, chunk_bytes, data_out.ctypes.data, data_out.size,
                                           meta_out.ctypes.data, meta_out.size, C.byref(res), C.byref(total), err, 512)
        if st != 0:
            raise YbGpuError(st, err.value.decode(errors="replace"))
        return data_out[:res.data_len], meta_out[:res.meta_len], res, total


class SstPiece(C.Structure):
    _fields_ = [("meta_file", C.c_void_p), ("meta_file_len", C.c_uint64), ("data_file_len", C.c_uint64),
                ("smallest_key", C.c_char_p), ("smallest_key_len", C.c_uint32),
                ("largest_key", C.c_char_p), ("largest_key_len", C.c_uint32)]


def sst_concat_meta(pieces, out=None, **table_kwargs):
    """ybgpu_sst_concat_meta. pieces: [(meta ndarray/bytes, data_len, smallest internal key, largest internal key)]
    in key order. Returns the metadata file (bytes; a view of `out` when a uint8 buffer is given) of the table
    whose data file is the pieces' data files back to back."""
    L = lib()
    L.ybgpu_sst_concat_meta.argtypes = [C.POINTER(JobOptions), C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    o, keep_o = make_options(**table_kwargs)
    arr = (SstPiece * len(pieces))()
    keep = []
    for i, (meta, data_len, smallest, largest) in enumerate(pieces):
        meta = np.ascontiguousarray(np.frombuffer(meta, np.uint8) if isinstance(meta, (bytes, bytearray)) else meta, dtype=np.uint8)
        keep += [meta, smallest, largest]
        arr[i] = SstPiece(meta.ctypes.data, meta.size, int(data_len), smallest, len(smallest), largest, len(largest))
    n = C.c_uint64()
    st = L.ybgpu_sst_concat_meta(C.byref(o), arr, len(pieces), None, 0, C.byref(n))
    if st != 0:
        raise YbGpuError(st, L.ybgpu_last_error().decode())
    buf = out if out is not None and out.size >= n.value else np.empty(n.value, np.uint8)
    st = L.ybgpu_sst_concat_meta(C.byref(o), arr, len(pieces), buf.ctypes.data, buf.size, C.byref(n))
    if st != 0:
        raise YbGpuError(st, L.ybgpu_last_error().decode())
    return buf[:n.value] if out is not None else buf[:n.value].tobytes()


def sst_check_supported(meta, data):
    """ybgpu_sst_check_supported: (status name, [blocks per CompressionType 0..7]) — host-side routing pre-check of one table."""
    L = lib()
    L.ybgpu_sst_check_supported.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64 * 8)]
    meta = np.ascontiguousarray(np.frombuffer(meta, np.uint8) if isinstance(meta, (bytes, bytearray)) else meta, dtype=np.uint8)
    data = np.ascontiguousarray(np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray)) else data, dtype=np.uint8)
    counts = (C.c_uint64 * 8)()
    st = L.ybgpu_sst_check_supported(meta.ctypes.data, meta.size, data.ctypes.data if data.size else None, data.size, C.byref(counts))
    return STATUS_NAMES.get(st, str(st)), list(counts)


def sst_verify_blocks(meta, data, stride=1):
    """ybgpu_sst_verify_blocks: (blocks checked, bad blocks) — host-side CRC32C check of every stride-th data block."""
    L = lib()
    L.ybgpu_sst_verify_blocks.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    meta = np.ascontiguousarray(np.frombuffer(meta, np.uint8) if isinstance(meta, (bytes, bytearray)) else meta, dtype=np.uint8)
    data = np.ascontiguousarray(np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray)) else data, dtype=np.uint8)
    n, bad = C.c_uint64(), C.c_uint64()
    st = L.ybgpu_sst_verify_blocks(meta.ctypes.data, meta.size, data.ctypes.data, data.size, stride, C.byref(n), C.byref(bad))
    if st not in (0, 2):
        raise YbGpuError(st, L.ybgpu_last_error().decode())
    return n.value, bad.value


def sst_verify_device(meta, data, device=0):
    """ybgpu_sst_verify_device: checksums, compressed streams, every entry and the key order of a split SST, checked on
    the GPU. Returns the OutputCheck; raises OutputCheckError (Corruption, .check = the first failure) for a bad table."""
    L = lib()
    L.ybgpu_sst_verify_device.argtypes = [C.c_int32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(OutputCheck)]
    meta = np.ascontiguousarray(np.frombuffer(meta, np.uint8) if isinstance(meta, (bytes, bytearray)) else meta, dtype=np.uint8)
    data = np.ascontiguousarray(np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray)) else data, dtype=np.uint8)
    chk = OutputCheck()
    st = L.ybgpu_sst_verify_device(device, meta.ctypes.data, meta.size, data.ctypes.data if data.size else None, data.size, C.byref(chk))
    if st != 0:
        raise OutputCheckError(st, L.ybgpu_last_error().decode(), chk)
    return chk
