"""K5's conversions, exhaustively: every F32 bit pattern (2^32) through cvk_gather_cast into bfloat16 and float16, and every FP8 byte
times every 16-bit scale (all 65,536 bfloat16 and all 65,536 float16 patterns) and times every float32 exponent through
cvk_gather_cast_scaled, into float32, float16 and bfloat16.  A NaN only has to stay a NaN.

The F32 sweep runs in slices of 2^28 patterns made on the device and compares them there against torch's CUDA Tensor.to(), a
conversion independent of K5's integer rounding code; a sample of 2^24 patterns covering every sign and exponent first pins that
reference to torch (bfloat16) and numpy (float16) on the CPU.  The scaled sweeps compare against (x.float() * s.float()).to(dst) on
the CPU.  On the host-side stand-ins (tests/simt_emu) every sweep runs on a strided sample: every 4099th F32 pattern, one scale in 64."""
import numpy as np
import pytest

from curvine_b200 import _lib
from test_zzz_readv_cast_gpu import MOCK
from test_zzz_readv_scaled_gpu import _assert_same, _code

pytestmark = pytest.mark.gpu

F8 = ["float8_e4m3fn", "float8_e5m2"]
DSTS = ["float32", "float16", "bfloat16"]
F32_SLICE = 1 << 28
F32_STRIDE = 4099  # the stand-ins' sample of the F32 sweep
SCALE_STRIDE = 64  # and of the scale sweeps


def _torch():
    import torch
    return torch


def _k5(src, segs, total, dst_bytes, scales=None):
    """one launch of cvk_gather_cast (scales None) or cvk_gather_cast_scaled over device bytes `src` -> the destination bytes"""
    torch = _torch()
    from curvine_b200 import kernels as K
    dst = torch.empty(dst_bytes, dtype=torch.uint8, device=src.device)
    d_segs, n = K.cast_segs_to_device(segs, src.device)
    assert n == total
    before = K.launch_count()
    if scales is None:
        K.gather_cast(src, d_segs, len(segs), total, dst)
    else:
        K.gather_cast_scaled(src, d_segs, K.scale_segs_to_device(scales, src.device), len(segs), total, dst)
    assert K.launch_count() == before + 1
    return dst


def _f32_slices(torch, dev):
    """the F32 bit patterns in slices, as int32 tensors on `dev`: all 2^32 in 16 slices, or every F32_STRIDE-th on the stand-ins"""
    if MOCK:
        yield torch.from_numpy((np.arange(-(-(1 << 32) // F32_STRIDE), dtype=np.uint64) * F32_STRIDE).astype(np.uint32).view(np.int32))
        return
    base = torch.arange(F32_SLICE, dtype=torch.int32, device=dev)
    for k in range((1 << 32) // F32_SLICE):
        off = k * F32_SLICE
        yield base + (off if off < (1 << 31) else off - (1 << 32))  # stays inside int32: no wrap-around


@pytest.mark.parametrize("dst_name", ["bfloat16", "float16"])
def test_the_device_reference_agrees_with_the_cpu_on_every_exponent(cuda, dst_name):
    """2^24 patterns (2^18 on the stand-ins): every sign and exponent with the mantissas around each rounding edge and random ones.
    torch's CUDA .to() -- the sweep's reference -- and K5 both equal torch (bfloat16) or numpy (float16) on the CPU."""
    torch = _torch()
    ddt = getattr(torch, dst_name)
    per = (1 << 15) >> (6 if MOCK else 0)
    m = np.random.default_rng(41).integers(0, 1 << 23, size=(512, per), dtype=np.uint32)
    edges = [0, 1, 2, 0x7FFFFF, 0x7FFFFE, 0x400000, 0x400001, 0x3FFFFF, 0x8000, 0x7FFF, 0x8001, 0x18000, 0x1000, 0xFFF, 0x1001, 0x3000, 0x2000,
             0x6000, 0x5FFF, 0x6001, 0x7FE000, 0x7FF000, 0x7FEFFF, 0x7FF001]
    m[:, :len(edges)] = np.array(edges, dtype=np.uint32)
    bits = ((np.arange(512, dtype=np.uint32) << 23)[:, None] | m).reshape(-1)  # sign and exponent from the row
    x = torch.from_numpy(bits.view(np.float32))
    if ddt == torch.float16:
        with np.errstate(over="ignore", invalid="ignore"):
            cpu = torch.from_numpy(bits.view(np.float32).astype(np.float16))
    else:
        cpu = x.to(ddt)
    _assert_same(x.to(cuda).to(ddt).cpu(), cpu, "torch's device conversion")
    n = bits.size
    got = _k5(x.view(torch.uint8).to(cuda), [(0, 0, n, 1, 0, 0, _lib.DTYPE_F32, _code(ddt))], n, 2 * n)
    _assert_same(got.cpu().view(ddt), cpu, "K5")


@pytest.mark.parametrize("dst_name", ["bfloat16", "float16"])
def test_every_f32_pattern_converts_like_the_device_reference(cuda, dst_name):
    torch = _torch()
    ddt = getattr(torch, dst_name)
    seen = 0
    for x in _f32_slices(torch, cuda):
        n = x.numel()
        got = _k5(x.view(torch.uint8), [(0, 0, n, 1, 0, 0, _lib.DTYPE_F32, _code(ddt))], n, 2 * n)
        _assert_same(got.view(ddt), x.view(torch.float32).to(ddt), (dst_name, seen))
        seen += n
        del x, got
    assert seen == (-(-(1 << 32) // F32_STRIDE) if MOCK else 1 << 32)


def _scaled_sweep(cuda, src_name, dst_name, scale_bits, scale_dt):
    """every FP8 byte times every scale of `scale_bits` (int array of the scale dtype's bit patterns): a [len(scale_bits), 256] view
    with block_rows = 1 and block_cols = 256, so view row r holds the 256 FP8 patterns and takes scale r"""
    torch = _torch()
    sdt, ddt = getattr(torch, src_name), getattr(torch, dst_name)
    int_dt = {2: torch.int16, 4: torch.int32}[scale_dt.itemsize]
    s = torch.from_numpy(np.ascontiguousarray(scale_bits)).to(int_dt).view(scale_dt)
    rows = s.numel()
    n = rows * 256
    src = torch.arange(256, dtype=torch.int32).to(torch.uint8).repeat(rows)
    d_s = s.to(cuda)
    got = _k5(src.to(cuda), [(0, 0, n, 1, 0, 0, _code(sdt), _code(ddt))], n, n * ddt.itemsize,
              [(d_s.data_ptr(), _code(scale_dt), 1, 256, 1, 256, 0, 0)])
    x = torch.arange(256, dtype=torch.int32).to(torch.uint8).view(sdt).float()
    want = (x[None, :] * s.float()[:, None]).to(ddt).reshape(-1)
    _assert_same(got.cpu().view(ddt), want, (src_name, dst_name, str(scale_dt)))


@pytest.mark.parametrize("scale_name", ["bfloat16", "float16"])
@pytest.mark.parametrize("dst_name", DSTS)
@pytest.mark.parametrize("src_name", F8)
def test_every_fp8_byte_times_every_16_bit_scale(cuda, src_name, dst_name, scale_name):
    """65,536 scales (1,024 on the stand-ins; their sample still holds +-0, +-inf, the NaNs 0x7fc0 / 0x7e00 and the subnormals' edges)"""
    torch = _torch()
    bits = np.arange(0, 1 << 16, SCALE_STRIDE if MOCK else 1, dtype=np.int64).astype(np.uint16).view(np.int16)
    _scaled_sweep(cuda, src_name, dst_name, bits, getattr(torch, scale_name))


def _f32_scale_bits():
    """both signs x every exponent x the mantissas 0, 1, 0x400000, 0x7fffff and 32 seeded random ones: products that are subnormal in
    float32 and in the destination, that overflow, and infinite or NaN scales"""
    mant = np.concatenate([np.array([0, 1, 0x400000, 0x7FFFFF], dtype=np.uint32),
                           np.random.default_rng(43).integers(0, 1 << 23, size=32, dtype=np.uint32)])
    bits = ((np.arange(512, dtype=np.uint32) << 23)[:, None] | mant[None, :]).reshape(-1)
    return bits[::SCALE_STRIDE // 4 if MOCK else 1].view(np.int32)


@pytest.mark.parametrize("dst_name", DSTS)
@pytest.mark.parametrize("src_name", F8)
def test_every_fp8_byte_times_every_f32_exponent(cuda, src_name, dst_name):
    _scaled_sweep(cuda, src_name, dst_name, _f32_scale_bits(), _torch().float32)
