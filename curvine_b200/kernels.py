"""Thin Python handles on the cvk_* launchers (include/curvine_b200_kernels.h) for tests and bench.py.

torch is plumbing here (device memory + streams); every byte of work happens in libcurvine_b200.so.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from ._lib import CvCastSeg, CvFrameDesc, CvScaleSeg, CvSeg, CvStreamDesc, CvStridedSeg, check

POLY_IEEE, POLY_CASTAGNOLI = 0, 1


def _stream_ptr(stream=None):
    s = stream if stream is not None else torch.cuda.current_stream()
    return ctypes.c_void_p(s.cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _struct_array_to_device(arr, device):
    raw = np.frombuffer(bytes(arr), dtype=np.uint8).copy()
    return torch.from_numpy(raw).to(device)


def launch_count() -> int:
    return int(_lib.lib().cvk_launch_count())


def crc_blocks(data: torch.Tensor, offs, lens, poly=POLY_IEEE, stream=None, out=None, base_offset=0):
    """CRC of data[off:off+len] for each (off, len).  ``data`` is a uint8 CUDA tensor."""
    dev = data.device
    offs_t = offs if isinstance(offs, torch.Tensor) else torch.tensor(np.asarray(offs, dtype=np.uint64).view(np.int64), device=dev)
    lens_t = lens if isinstance(lens, torch.Tensor) else torch.tensor(np.asarray(lens, dtype=np.uint64).view(np.int64), device=dev)
    n = offs_t.numel()
    total = int(lens_t.sum().item())
    if out is None:
        out = torch.empty(n, dtype=torch.int32, device=dev)
    check(_lib.lib().cvk_crc_blocks(ctypes.c_void_p(data.data_ptr() + base_offset), _ptr(offs_t), _ptr(lens_t), n, poly,
                                    total, _ptr(out), _stream_ptr(stream)), "cvk_crc_blocks")
    return out


def crc_blocks_raw(data_ptr, offs_t, lens_t, n, poly, total, out, stream=None):
    check(_lib.lib().cvk_crc_blocks(ctypes.c_void_p(data_ptr), _ptr(offs_t), _ptr(lens_t), n, poly, total, _ptr(out),
                                    _stream_ptr(stream)), "cvk_crc_blocks")


def verify_crcs(crc, expect, n_bad, bad_mask=None, stream=None):
    check(_lib.lib().cvk_verify_crcs(_ptr(crc), _ptr(expect), crc.numel(), _ptr(n_bad), _ptr(bad_mask),
                                     _stream_ptr(stream)), "cvk_verify_crcs")


def frame_descs_to_device(descs, device):
    arr = (CvFrameDesc * len(descs))(*descs)
    return _struct_array_to_device(arr, device)


def stream_descs_to_device(descs, device):
    arr = (CvStreamDesc * len(descs))(*descs)
    return _struct_array_to_device(arr, device)


def segs_to_device(segs, device):
    arr = (CvSeg * len(segs))(*[CvSeg(*s) for s in segs])
    return _struct_array_to_device(arr, device)


def unpack_frames(wire, d_desc, n_frames, n_blocks, dst, poly, total_bytes, want_crc=True, want_err=True, stream=None):
    dev = wire.device
    crc = torch.empty(n_blocks, dtype=torch.int32, device=dev) if want_crc else None
    err = torch.empty(n_frames, dtype=torch.int32, device=dev) if want_err else None
    check(_lib.lib().cvk_unpack_frames(_ptr(wire), _ptr(d_desc), n_frames, n_blocks, _ptr(dst), poly, total_bytes,
                                       _ptr(crc), _ptr(err), _stream_ptr(stream)), "cvk_unpack_frames")
    return crc, err


def expand_streams(d_streams, n_streams, n_frames, device, stream=None):
    out = torch.empty(n_frames * ctypes.sizeof(CvFrameDesc), dtype=torch.uint8, device=device)
    check(_lib.lib().cvk_expand_streams(_ptr(d_streams), n_streams, _ptr(out), n_frames, _stream_ptr(stream)),
          "cvk_expand_streams")
    return out


def pack_frames(src, d_desc, n_frames, n_blocks, wire, poly, total_bytes, want_crc=True, stream=None):
    crc = torch.empty(n_blocks, dtype=torch.int32, device=src.device) if want_crc else None
    check(_lib.lib().cvk_pack_frames(_ptr(src), _ptr(d_desc), n_frames, n_blocks, _ptr(wire), poly, total_bytes,
                                     _ptr(crc), _stream_ptr(stream)), "cvk_pack_frames")
    return crc


def gather_pages(src, d_segs, n, total_bytes, dst, stream=None):
    check(_lib.lib().cvk_gather_pages(_ptr(src), _ptr(d_segs), n, total_bytes, _ptr(dst), _stream_ptr(stream)),
          "cvk_gather_pages")


def strided_segs_to_device(segs, device):
    """segs: list of (src_off, dst_off, len, rows, src_pitch, dst_pitch)"""
    arr = (CvStridedSeg * len(segs))(*[CvStridedSeg(*s) for s in segs])
    return _struct_array_to_device(arr, device)


def gather_strided(src, d_segs, n, total_bytes, dst, stream=None):
    check(_lib.lib().cvk_gather_strided(_ptr(src), _ptr(d_segs), n, total_bytes, _ptr(dst), _stream_ptr(stream)),
          "cvk_gather_strided")


def cast_segs_to_device(segs, device):
    """segs: list of (src_off, dst_off, elems, rows, src_pitch, dst_pitch, src_dtype, dst_dtype) with _lib.DTYPE_* codes; `first` (the
    work distribution) is filled here.  -> (device table, total elements)"""
    arr = (CvCastSeg * len(segs))()
    first = total = 0
    for i, (so, do, elems, rows, sp, dp, sdt, ddt) in enumerate(segs):
        arr[i] = CvCastSeg(so, do, elems, rows, sp, dp, first, sdt, ddt)
        first += rows * _lib.cast_row_chunks(elems)
        total += elems * rows
    return _struct_array_to_device(arr, device), total


def gather_cast(src, d_segs, n, total_elems, dst, stream=None):
    check(_lib.lib().cvk_gather_cast(_ptr(src), _ptr(d_segs), n, total_elems, _ptr(dst), _stream_ptr(stream)), "cvk_gather_cast")


def scale_segs_to_device(scales, device):
    """scales: one entry per cast segment, None (not scaled) or (scale_ptr, scale_dtype, block_rows, block_cols, scale_cols, cols, view0,
    view_step) with a _lib.DTYPE_* scale dtype (see CvScaleSeg).  -> device table"""
    arr = (CvScaleSeg * len(scales))()
    for i, sc in enumerate(scales):
        if sc is not None:
            ptr, dt, br, bc, scols, cols, view0, step = sc
            arr[i] = CvScaleSeg(ptr, br, bc, scols, cols, view0, step, dt, 0)
    return _struct_array_to_device(arr, device)


def gather_cast_scaled(src, d_segs, d_scales, n, total_elems, dst, stream=None):
    check(_lib.lib().cvk_gather_cast_scaled(_ptr(src), _ptr(d_segs), _ptr(d_scales), n, total_elems, _ptr(dst), _stream_ptr(stream)),
          "cvk_gather_cast_scaled")


def deinterleave_blocks(gathered, shard_stride, world, block_size, n_blocks, file_len, dst, stream=None):
    check(_lib.lib().cvk_deinterleave_blocks(_ptr(gathered), shard_stride, world, block_size, n_blocks, file_len,
                                             _ptr(dst), _stream_ptr(stream)), "cvk_deinterleave_blocks")


def gather_shards_p2p(shard_ptrs, block_size, n_blocks, file_len, dst, stream=None):
    """shard_ptrs: list of device pointers (ints), one per rank, local or peer-mapped."""
    arr = (ctypes.c_uint64 * len(shard_ptrs))(*shard_ptrs)
    check(_lib.lib().cvk_gather_shards_p2p(arr, len(shard_ptrs), block_size, n_blocks, file_len, _ptr(dst), _stream_ptr(stream)),
          "cvk_gather_shards_p2p")


def u32(t: torch.Tensor) -> np.ndarray:
    """int32 CUDA tensor -> uint32 numpy."""
    return t.cpu().numpy().view(np.uint32)
