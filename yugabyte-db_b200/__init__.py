"""yugabyte-db_b200 — H100-native DocDB compaction engine.

Python is only the test / bench binding over the C ABI in include/ybgpu_compaction.h (the product
is libybgpu.so: hand-written sm_90a CUDA + a C++ host layer). Importing this package never
falls back to a CPU implementation: if libybgpu.so is missing the import fails loudly.
"""
from .binding import (  # noqa: F401
    GpuCompactionJob, JobOptions, JobStats, BlockHandle, YbGpuError, lib, device_count,
    HT_MIN, HT_MAX, HT_INVALID, TTL_MAX_NS, MAX_SEQUENCE, LIB_PATH, HostTableBuilder, GenConfig, GeneratedSst, generate_ssts, PHASE_NAMES, sst_block_handles, sst_separators,
    compact_files, plan_subcompactions, sst_last_key, make_options, STREAM_PRIVATE, InputFile, SubOutput, sst_concat_meta, SstPiece, sst_verify_blocks, sst_check_supported, STATUS_NAMES, bind_thread_to_device, compact_files_one_table, OneTableResult, RangeComm, RangeShardResult, range_comm_unique_id, generate_sst_files, PATH_FUSED_INGEST, PATH_GENERAL_DECODE, PATH_SNAPPY, PATH_PARTITION_RETRY, PATH_ENCODER_V4, PATH_ENCODER_V5, PATH_KV_INPUT, PATH_SNAPPY_OUTPUT,
    PATH_LZ4, PATH_LZ4_OUTPUT, PATH_INGEST_RETRY, PATH_FAST_DECODE, PATH_ENCODER_FUSED, COMPRESSION_NONE, COMPRESSION_SNAPPY, COMPRESSION_LZ4,
    PATH_OUTPUT_VERIFIED, OutputCheck, OutputCheckError, CHECK_KIND_NAMES, sst_verify_device, split_range, sst_uncompressed_bytes,
)
