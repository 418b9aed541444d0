"""ctypes loader for libcurvine_b200.so (the C-ABI drop-in boundary).

Fails loudly: there is no CPU or PyTorch fallback for any entry point.
"""
import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libcurvine_b200.so")

_lib = None


class CvFrameDesc(ctypes.Structure):
    _fields_ = [("wire_off", ctypes.c_uint64), ("dst_off", ctypes.c_uint64), ("data_len", ctypes.c_uint32),
                ("header_len", ctypes.c_uint32), ("req_id", ctypes.c_int64), ("seq_id", ctypes.c_int32),
                ("block", ctypes.c_uint32), ("code", ctypes.c_uint8), ("status", ctypes.c_uint8),
                ("pad_", ctypes.c_uint8 * 2), ("tail_clip", ctypes.c_uint32)]


class CvStreamDesc(ctypes.Structure):
    _fields_ = [("wire_off", ctypes.c_uint64), ("dst_off", ctypes.c_uint64), ("block_len", ctypes.c_uint64),
                ("req_id", ctypes.c_int64), ("chunk_size", ctypes.c_uint32), ("first_seq_id", ctypes.c_int32),
                ("block", ctypes.c_uint32), ("first_frame", ctypes.c_uint32), ("code", ctypes.c_uint8),
                ("status", ctypes.c_uint8), ("pad_", ctypes.c_uint8 * 2), ("tail_clip", ctypes.c_uint32)]


class CvSeg(ctypes.Structure):
    _fields_ = [("src_off", ctypes.c_uint64), ("dst_off", ctypes.c_uint64), ("len", ctypes.c_uint64)]


class CvRange(ctypes.Structure):
    _fields_ = [("file_off", ctypes.c_int64), ("len", ctypes.c_int64), ("d_dst", ctypes.c_void_p)]


class CvStridedRange(ctypes.Structure):
    _fields_ = [("file_off", ctypes.c_int64), ("row_len", ctypes.c_int64), ("rows", ctypes.c_int64), ("file_pitch", ctypes.c_int64),
                ("d_dst", ctypes.c_void_p), ("dst_pitch", ctypes.c_int64)]


class CvStridedSeg(ctypes.Structure):
    _fields_ = [("src_off", ctypes.c_uint64), ("dst_off", ctypes.c_uint64), ("len", ctypes.c_uint64), ("rows", ctypes.c_uint64),
                ("src_pitch", ctypes.c_uint64), ("dst_pitch", ctypes.c_uint64)]


class CvCastRange(ctypes.Structure):
    _fields_ = CvStridedRange._fields_ + [("src_dtype", ctypes.c_int32), ("dst_dtype", ctypes.c_int32)]


class CvCastSeg(ctypes.Structure):
    _fields_ = [("src_off", ctypes.c_uint64), ("dst_off", ctypes.c_uint64), ("elems", ctypes.c_uint64), ("rows", ctypes.c_uint64),
                ("src_pitch", ctypes.c_uint64), ("dst_pitch", ctypes.c_uint64), ("first", ctypes.c_uint64), ("src_dtype", ctypes.c_int32),
                ("dst_dtype", ctypes.c_int32)]


class CvScaleSeg(ctypes.Structure):
    _fields_ = [("scale", ctypes.c_void_p), ("block_rows", ctypes.c_uint64), ("block_cols", ctypes.c_uint64), ("scale_cols", ctypes.c_uint64),
                ("cols", ctypes.c_uint64), ("view0", ctypes.c_uint64), ("view_step", ctypes.c_uint64), ("scale_dtype", ctypes.c_int32),
                ("pad", ctypes.c_int32)]


class CvScaledRange(ctypes.Structure):
    _fields_ = [("cast", CvCastRange), ("d_scale", ctypes.c_void_p), ("scale_dtype", ctypes.c_int32), ("pad", ctypes.c_int32),
                ("scale_rows", ctypes.c_int64), ("scale_cols", ctypes.c_int64), ("block_rows", ctypes.c_int64), ("block_cols", ctypes.c_int64),
                ("cols", ctypes.c_int64), ("first_elem", ctypes.c_int64)]


# include/curvine_b200_kernels.h: element types of cast reads and cvk_gather_cast (the two FP8 codes: sources only)
DTYPE_NONE, DTYPE_F32, DTYPE_F16, DTYPE_BF16, DTYPE_F8_E4M3, DTYPE_F8_E5M2 = 0, 1, 2, 3, 4, 5
FLOAT_CODES = (DTYPE_F32, DTYPE_F16, DTYPE_BF16)  # conversion targets and scale dtypes
F8_CODES = (DTYPE_F8_E4M3, DTYPE_F8_E5M2)  # sources only


def cast_row_chunks(elems: int) -> int:
    """CV_CAST_ROW_CHUNKS: work chunks of one row of a CvCastSeg"""
    return (elems + 14) // 8 if elems else 0


assert ctypes.sizeof(CvStridedRange) == 48 and ctypes.sizeof(CvStridedSeg) == 48
assert ctypes.sizeof(CvCastRange) == 56 and ctypes.sizeof(CvCastSeg) == 64
assert ctypes.sizeof(CvScaledRange) == 120 and ctypes.sizeof(CvScaleSeg) == 64
assert ctypes.sizeof(CvFrameDesc) == 48 and ctypes.sizeof(CvStreamDesc) == 56 and ctypes.sizeof(CvSeg) == 24 and ctypes.sizeof(CvRange) == 24


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError("%s is missing: run `python -m curvine_b200.build` (needs nvcc); "
                              "curvine_b200 has no CPU fallback" % LIB_PATH)
        _lib = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
        _declare(_lib)
    return _lib


def _declare(L):
    vp, u8p, u32, u64, i = ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_int
    L.cvk_init.argtypes, L.cvk_init.restype = [i], i
    L.cvk_launch_count.argtypes, L.cvk_launch_count.restype = [], u64
    sz, vpp = ctypes.c_size_t, ctypes.POINTER(ctypes.c_void_p)
    L.cvh_pinned_alloc.argtypes, L.cvh_pinned_alloc.restype = [sz, vpp], i
    L.cvh_device_alloc.argtypes, L.cvh_device_alloc.restype = [sz, vpp], i
    L.cvh_pinned_free.argtypes, L.cvh_pinned_free.restype = [vp], i
    L.cvh_host_register.argtypes, L.cvh_host_register.restype = [vp, sz], i
    L.cvh_host_unregister.argtypes, L.cvh_host_unregister.restype = [vp], i
    L.cvh_device_free.argtypes, L.cvh_device_free.restype = [vp], i
    L.cvh_h2d_async.argtypes, L.cvh_h2d_async.restype = [vp, vp, sz, vp, vp], i
    L.cvh_d2h_async.argtypes, L.cvh_d2h_async.restype = [vp, vp, sz, vp, vp], i
    L.cvh_stream_create.argtypes, L.cvh_stream_create.restype = [vpp], i
    L.cvh_event_create.argtypes, L.cvh_event_create.restype = [vpp], i
    for name in ("cvh_stream_destroy", "cvh_stream_synchronize", "cvh_event_destroy", "cvh_event_synchronize", "cvh_event_query"):
        getattr(L, name).argtypes, getattr(L, name).restype = [vp], i
    L.cvh_stream_wait_event.argtypes, L.cvh_stream_wait_event.restype = [vp, vp], i
    L.cvh_event_record.argtypes, L.cvh_event_record.restype = [vp, vp], i
    L.cvk_tune.argtypes, L.cvk_tune.restype = [i, i], i
    L.cvk_profile_enable.argtypes, L.cvk_profile_enable.restype = [i], i
    L.cvk_profile_collect.argtypes, L.cvk_profile_collect.restype = [ctypes.POINTER(ctypes.c_double), ctypes.POINTER(u32)], i
    L.cvk_crc_blocks.argtypes, L.cvk_crc_blocks.restype = [u8p, vp, vp, u32, i, u64, vp, vp], i
    L.cvk_verify_crcs.argtypes, L.cvk_verify_crcs.restype = [vp, vp, u32, vp, vp, vp], i
    L.cvk_verify_crcs_masked.argtypes, L.cvk_verify_crcs_masked.restype = [vp, vp, vp, u32, vp, vp, vp], i
    L.cvk_unpack_frames.argtypes, L.cvk_unpack_frames.restype = [u8p, vp, u32, u32, u8p, i, u64, vp, vp, vp], i
    L.cvk_expand_streams.argtypes, L.cvk_expand_streams.restype = [vp, u32, vp, u32, vp], i
    L.cvk_gather_pages.argtypes, L.cvk_gather_pages.restype = [u8p, vp, u32, u64, u8p, vp], i
    L.cvk_gather_strided.argtypes, L.cvk_gather_strided.restype = [u8p, vp, u32, u64, u8p, vp], i
    L.cvk_gather_cast.argtypes, L.cvk_gather_cast.restype = [u8p, vp, u32, u64, u8p, vp], i
    L.cvk_gather_cast_scaled.argtypes, L.cvk_gather_cast_scaled.restype = [u8p, vp, vp, u32, u64, u8p, vp], i
    L.cvk_pack_frames.argtypes, L.cvk_pack_frames.restype = [u8p, vp, u32, u32, u8p, i, u64, vp, vp], i
    L.cvk_deinterleave_blocks.argtypes = [u8p, u64, u32, u64, u64, u64, u8p, vp]
    L.cvk_deinterleave_blocks.restype = i
    L.cvk_gather_shards_p2p.argtypes, L.cvk_gather_shards_p2p.restype = [vp, u32, u64, u64, u64, u8p, vp], i
    # ---- upper boundary (include/curvine_b200.h)
    c, i64, i32, cp = ctypes.c_char_p, ctypes.c_int64, ctypes.c_int32, ctypes.POINTER
    L.cv_last_error.argtypes, L.cv_last_error.restype = [], c
    L.cv_free.argtypes, L.cv_free.restype = [vp], None
    L.cv_fs_new.argtypes, L.cv_fs_new.restype = [c, cp(vp)], i64
    L.cv_fs_new_from_string.argtypes, L.cv_fs_new_from_string.restype = [c, cp(vp)], i64
    L.cv_fs_load_namespace.argtypes, L.cv_fs_load_namespace.restype = [vp, c], i64
    L.cv_fs_load_namespace_string.argtypes, L.cv_fs_load_namespace_string.restype = [vp, c], i64
    L.cv_fs_close.argtypes, L.cv_fs_close.restype = [vp], i64
    L.cv_fs_wait_registered.argtypes, L.cv_fs_wait_registered.restype = [vp], i64
    L.cv_fs_preregister.argtypes, L.cv_fs_preregister.restype = [vp], i64
    L.cv_fs_arena_stats.argtypes, L.cv_fs_arena_stats.restype = [vp, cp(u64)], i64
    L.cv_synth_delete_file.argtypes, L.cv_synth_delete_file.restype = [vp, i64, i64], i64
    L.cv_worker_arena_stats.argtypes, L.cv_worker_arena_stats.restype = [vp, cp(i64)], i64
    L.cv_gds_info.argtypes, L.cv_gds_info.restype = [cp(i64)], i64
    L.cv_gpu_numa_node.argtypes, L.cv_gpu_numa_node.restype = [i32], i64
    L.cv_fs_metrics.argtypes, L.cv_fs_metrics.restype = [vp, cp(i64)], i64
    L.cv_fs_pool_stats.argtypes, L.cv_fs_pool_stats.restype = [vp, cp(i64)], i64
    L.cv_open.argtypes, L.cv_open.restype = [vp, c, cp(vp), cp(i64)], i64
    L.cv_read.argtypes, L.cv_read.restype = [vp, cp(vp), cp(i64)], i64
    L.cv_read_buf.argtypes, L.cv_read_buf.restype = [vp, vp, i64, cp(i64)], i64
    L.cv_read_full.argtypes, L.cv_read_full.restype = [vp, vp, i64, cp(i64)], i64
    L.cv_fuse_read.argtypes = [vp, i64, i64, vp, cp(i64), cp(i64), i32, cp(i32)]
    L.cv_fuse_read.restype = i64
    L.cv_seek.argtypes, L.cv_seek.restype = [vp, i64], i64
    L.cv_pos.argtypes, L.cv_pos.restype = [vp], i64
    L.cv_len.argtypes, L.cv_len.restype = [vp], i64
    L.cv_chunk_size.argtypes, L.cv_chunk_size.restype = [vp], i64
    L.cv_close_reader.argtypes, L.cv_close_reader.restype = [vp], i64
    L.cv_read_device.argtypes, L.cv_read_device.restype = [vp, vp, i64, vp, cp(i64)], i64
    L.cv_read_device_sharded.argtypes = [vp, i32, i32, vp, i64, vp, cp(i64)]
    L.cv_read_device_sharded.restype = i64
    L.cv_read_many_device.argtypes = [vp, cp(c), i32, vp, vp, i64, vp, cp(u64), cp(u32), cp(u64), cp(i64)]
    L.cv_read_many_device.restype = i64
    L.cv_shard_plan.argtypes = [vp, i32, i32, vp, vp, vp, vp, i32, cp(i32), cp(i64)]
    L.cv_shard_plan.restype = i64
    L.cv_readv_device.argtypes, L.cv_readv_device.restype = [vp, cp(CvRange), i32, vp, cp(i64)], i64
    L.cv_readv_plan.argtypes = [vp, cp(CvRange), i32, cp(i64), cp(i64), cp(i64), cp(i32), cp(i32), i32, cp(i32), cp(i64), cp(i64)]
    L.cv_readv_plan.restype = i64
    L.cv_readv_strided_device.argtypes, L.cv_readv_strided_device.restype = [vp, cp(CvStridedRange), i32, vp, cp(i64)], i64
    L.cv_readv_strided_plan.argtypes = [vp, cp(CvStridedRange), i32, cp(i64), cp(i64), cp(i64), cp(i64), cp(i32), cp(i32), i32, cp(i32), cp(i64),
                                        cp(i64)]
    L.cv_readv_strided_plan.restype = i64
    L.cv_readv_cast_device.argtypes, L.cv_readv_cast_device.restype = [vp, cp(CvCastRange), i32, vp, cp(i64)], i64
    L.cv_readv_scaled_device.argtypes, L.cv_readv_scaled_device.restype = [vp, cp(CvScaledRange), i32, vp, cp(i64)], i64
    L.cv_readv_cast_plan.argtypes = [vp, cp(CvCastRange), i32, cp(i64), cp(i64), cp(i64), cp(i64), cp(i32), cp(i32), i32, cp(i32), cp(i64), cp(i64)]
    L.cv_readv_cast_plan.restype = i64
    L.cv_fuse_read_device.argtypes = [vp, i64, i64, vp, vp, vp, i32, i64, vp, cp(i64)]
    L.cv_fuse_read_device.restype = i64
    L.cv_fuse_read_file_device.argtypes = [vp, c, i64, vp, vp, vp, i32, i64, vp, cp(i64), cp(u32)]
    L.cv_fuse_read_file_device.restype = i64
    L.cv_verify.argtypes, L.cv_verify.restype = [vp, cp(u64), cp(u32), cp(u64)], i64
    L.cv_device_stats.argtypes, L.cv_device_stats.restype = [vp, cp(CvReadStats)], i64
    L.cv_writer_open.argtypes, L.cv_writer_open.restype = [vp, c, i64, i64, i32, c, i32, i64, cp(vp)], i64
    L.cv_write.argtypes, L.cv_write.restype = [vp, vp, i64], i64
    L.cv_write_device.argtypes, L.cv_write_device.restype = [vp, vp, i64, vp], i64
    L.cv_writer_close.argtypes, L.cv_writer_close.restype = [vp, i32, cp(vp)], i64
    L.cv_worker_start.argtypes, L.cv_worker_start.restype = [c, cp(vp), cp(i32)], i64
    L.cv_worker_stop.argtypes, L.cv_worker_stop.restype = [vp], i64
    L.cv_worker_hbm_load.argtypes, L.cv_worker_hbm_load.restype = [vp, i64, i32], i64
    L.cv_worker_hbm_drain.argtypes, L.cv_worker_hbm_drain.restype = [vp], i64
    L.cv_worker_hbm_stats.argtypes, L.cv_worker_hbm_stats.restype = [vp, cp(i64)], i64
    L.cv_worker_hbm_tier.argtypes, L.cv_worker_hbm_tier.restype = [vp, cp(i64)], i64
    L.cv_worker_metrics.argtypes, L.cv_worker_metrics.restype = [vp, cp(i64)], i64
    L.cv_synth_create_file.argtypes = [vp, c, i64, i64, i64, i32, i32, i32, i32, c, cp(vp)]
    L.cv_synth_create_file.restype = i64
    L.cv_synth_set_shard_world.argtypes, L.cv_synth_set_shard_world.restype = [i32], i64
    L.cv_synth_block.argtypes, L.cv_synth_block.restype = [u64, u64, vp, ctypes.c_size_t], None
    L.cv_host_crc.argtypes, L.cv_host_crc.restype = [i, vp, ctypes.c_size_t], u32


class CvReadStats(ctypes.Structure):
    _fields_ = [("bytes", ctypes.c_uint64), ("blocks", ctypes.c_uint64), ("verified", ctypes.c_uint64),
                ("h2d_bytes", ctypes.c_uint64), ("kernel_launches", ctypes.c_uint64), ("fetch_sec", ctypes.c_double),
                ("wall_sec", ctypes.c_double), ("reg_hits", ctypes.c_uint64), ("reg_misses", ctypes.c_uint64),
                ("ring_alloc_sec", ctypes.c_double), ("reg_rejected", ctypes.c_uint64), ("reg_bytes", ctypes.c_uint64),
                ("gds_bytes", ctypes.c_uint64)]


# every symbol include/*.h declares (tests check the .so exports all of them)
EXPORTS = ["cvk_init", "cvk_crc_blocks", "cvk_verify_crcs", "cvk_verify_crcs_masked", "cvk_unpack_frames", "cvk_expand_streams", "cvk_gather_pages",
           "cvk_gather_strided", "cvk_gather_cast", "cvk_gather_cast_scaled", "cvk_pack_frames", "cvk_deinterleave_blocks", "cvk_gather_shards_p2p", "cvk_launch_count", "cvk_tune", "cvk_profile_enable", "cvk_profile_collect", "cv_last_error", "cv_free", "cv_fs_new",
           "cv_fs_new_from_string", "cv_fs_load_namespace", "cv_fs_load_namespace_string", "cv_fs_close", "cv_fs_wait_registered", "cv_fs_preregister", "cv_fs_arena_stats", "cv_synth_delete_file", "cv_worker_arena_stats", "cv_gpu_numa_node", "cv_gds_info", "cv_fs_metrics", "cv_fs_pool_stats",
           "cv_open", "cv_read", "cv_read_buf", "cv_read_full", "cv_fuse_read", "cv_seek", "cv_pos", "cv_len",
           "cv_chunk_size", "cv_close_reader", "cv_read_device", "cv_read_device_sharded", "cv_read_many_device", "cv_shard_plan", "cv_readv_device", "cv_readv_plan", "cv_readv_strided_device", "cv_readv_strided_plan", "cv_readv_cast_device", "cv_readv_cast_plan", "cv_readv_scaled_device", "cv_fuse_read_device", "cv_fuse_read_file_device",
           "cv_verify", "cv_device_stats", "cv_writer_open", "cv_write", "cv_write_device", "cv_writer_close", "cv_worker_start", "cv_worker_stop", "cv_worker_hbm_load", "cv_worker_hbm_drain", "cv_worker_hbm_stats", "cv_worker_hbm_tier", "cv_worker_metrics",
           "cv_synth_create_file", "cv_synth_set_shard_world", "cv_synth_block", "cv_host_crc",
           "cvh_pinned_alloc", "cvh_pinned_free", "cvh_host_register", "cvh_host_unregister", "cvh_device_alloc", "cvh_device_free", "cvh_h2d_async", "cvh_d2h_async", "cvh_stream_create", "cvh_stream_destroy",
           "cvh_stream_synchronize", "cvh_stream_wait_event", "cvh_event_create", "cvh_event_destroy", "cvh_event_record", "cvh_event_synchronize", "cvh_event_query"]


class CudaError(RuntimeError):
    pass


def check(rc: int, what: str = ""):
    if rc != 0:
        raise CudaError("%s failed: cudaError %d" % (what or "cvk call", rc))
