"""FP8 checkpoints on load, on the GPU: K5's scaled instance (cvk_gather_cast_scaled) bit-exact against torch on the CPU -- every FP8
bit pattern unscaled, and (x.float() * s.float()).to(dst) with per-element scales --, scaled reads through the reader
(cv_readv_scaled_device) in every read mode mixed with unscaled FP8, plain-cast and plain ranges, its validation, and
safetensors.load_file(dtype=..., scales=..., scale_block=...) on a written FP8 checkpoint.  Runs on the host-side stand-ins too
(tests/simt_emu), where "device memory" is host memory."""
import ctypes

import numpy as np
import pytest

from curvine_b200 import _lib
from curvine_b200 import fs as F
from curvine_b200 import safetensors as ST
from oracle import clib, layout, synth
from test_zzz_readv_cast_gpu import BS, GUARD, MODES, MOCK, _conf, _flip, _fs_for, cluster  # noqa: F401  (cluster: a fixture)

pytestmark = pytest.mark.gpu


def _torch():
    import torch
    return torch


def _code(dt):
    torch = _torch()
    return {torch.float32: _lib.DTYPE_F32, torch.float16: _lib.DTYPE_F16, torch.bfloat16: _lib.DTYPE_BF16,
            torch.float8_e4m3fn: _lib.DTYPE_F8_E4M3, torch.float8_e5m2: _lib.DTYPE_F8_E5M2}[dt]


def _int_view(dt):
    torch = _torch()
    return {4: torch.int32, 2: torch.int16}[dt.itemsize]


def _assert_same(got, want, what=""):
    """got == want bit for bit, except that a NaN only has to stay a NaN"""
    torch = _torch()
    nan = torch.isnan(want.float())
    bad = (got.view(_int_view(want.dtype)) != want.view(_int_view(want.dtype))) & ~nan
    assert not bool(bad.any()), (what, int(bad.sum()), got[bad][:8], want[bad][:8])
    assert bool(torch.isnan(got.float()[nan]).all()), what


def _view(raw, dt):
    torch = _torch()
    return torch.from_numpy(np.array(raw, dtype=np.uint8)).view(dt)


def _scales(rng, n, dt):
    """n scales in dtype dt: random magnitudes 2^-40 .. 2^40 of both signs, and the edges -- zeros of both signs, scales whose
    products are denormal or overflow even in float32, exact powers of two"""
    torch = _torch()
    s = np.ldexp(rng.uniform(0.5, 1.0, n), rng.integers(-40, 41, n)) * np.where(rng.random(n) < 0.3, -1.0, 1.0)
    edge = [0.0, -0.0, 1.0, 2.0 ** -126, 2.0 ** -133, 3e-39, 2.0 ** 120, -2.0 ** 127, 1.0 / 448, 2.0 ** -16, 65504.0, 3.0e38]
    k = rng.choice(n, size=min(n, len(edge) * 2), replace=False)
    s[k] = np.resize(edge, k.size)
    return torch.from_numpy(s).to(dt)


def _reference(x, s_flat, idx, ddt):
    """torch on the CPU: (x.float() * s.float()).to(ddt), s being the scale each element takes"""
    return (x.float() * s_flat.float()[idx]).to(ddt)


def _scaled_on_device(cuda, src_bytes, segs, scales, dst_len):
    """cvk_gather_cast_scaled over uint8 `src_bytes` into a guard-filled buffer -> its bytes (numpy)"""
    torch = _torch()
    from curvine_b200 import kernels as K
    d_src = torch.from_numpy(np.ascontiguousarray(src_bytes)).to(cuda)
    dst = torch.full((dst_len,), GUARD, dtype=torch.uint8, device=cuda)
    d_segs, total = K.cast_segs_to_device(segs, cuda)
    d_scales = K.scale_segs_to_device(scales, cuda)
    K.gather_cast_scaled(d_src, d_segs, d_scales, len(segs), total, dst)
    torch.cuda.synchronize()
    return dst.cpu().numpy()


F8 = ["float8_e4m3fn", "float8_e5m2"]
DSTS = ["float32", "float16", "bfloat16"]


# ---- the kernel

@pytest.mark.parametrize("dst_name", DSTS)
@pytest.mark.parametrize("src_name", F8)
def test_every_fp8_pattern_converts_exactly(cuda, src_name, dst_name):
    """all 256 bit patterns, unscaled, at every source offset 0..8 (whole chunks read as one 8-byte load or bytewise)"""
    torch = _torch()
    sdt, ddt = getattr(torch, src_name), getattr(torch, dst_name)
    raw = np.concatenate([np.arange(256, dtype=np.uint8)] * 9)
    segs = [(k * 256 + k, k * 256 * ddt.itemsize + 64 * k, 256 - k, 1, 0, 0, _code(sdt), _code(ddt)) for k in range(9)]
    got = _scaled_on_device(cuda, raw, segs, [None] * len(segs), 9 * 256 * ddt.itemsize + 64 * 9)
    for so, do, n, _, _, _, _, _ in segs:
        _assert_same(_view(got[do:do + n * ddt.itemsize], ddt), _view(raw[so:so + n], sdt).to(ddt), (src_name, dst_name, so))


def _rect_case(cuda, rng, sdt, ddt, scale_dt, R, C, br, bc, n_seg):
    """an R x C FP8 weight at an odd offset, its block scales, and n_seg segments: rectangles of it (rows with the weight's pitch) and
    runs of whole rows as one long row (chunks that cross view rows), each landing at an element-aligned offset with guards between
    rows -> (src bytes, weight offset, segs, scales, dst_len, [(dst offset, dst_pitch, view indices per row)], scales on the CPU and
    on the device, scale grid shape)"""
    torch = _torch()
    base = int(rng.integers(1, 16))
    src = rng.integers(0, 256, size=base + R * C + 32, dtype=np.uint8)
    SR, SC = -(-R // br), -(-C // bc)
    s = _scales(rng, SR * SC, scale_dt)
    d_s = s.to(cuda)
    ds = ddt.itemsize
    segs, scales, where, at = [], [], [], 16
    for k in range(n_seg):
        if k % 3 == 2:  # a run of whole rows as one row
            r0 = int(rng.integers(0, R))
            c0 = int(rng.integers(0, C))
            n = int(rng.integers(1, (R - r0) * C - c0 + 1))
            v0, rows, elems, pitch = r0 * C + c0, 1, n, 0
        else:
            r0, c0 = int(rng.integers(0, R)), int(rng.integers(0, C))
            rows, elems = int(rng.integers(1, R - r0 + 1)), int(rng.integers(1, C - c0 + 1))
            v0, pitch = r0 * C + c0, C
        at += (-at) % ds + ds * int(rng.integers(0, 8))
        dp = elems * ds + ds * int(rng.integers(1, 6))
        segs.append((base + v0, at, elems, rows, pitch, dp, _code(sdt), _code(ddt)))
        scales.append((d_s.data_ptr(), _code(scale_dt), br, bc, SC, C, v0, pitch))
        where.append((at, dp, [np.arange(v0 + i * pitch, v0 + i * pitch + elems) for i in range(rows)]))
        at += rows * dp + 16
    return src, base, segs, scales, at + 64, where, s, d_s, (SR, SC)


@pytest.mark.parametrize("scale_name", ["float32", "bfloat16", "float16"])
@pytest.mark.parametrize("dst_name", DSTS)
@pytest.mark.parametrize("src_name", F8)
def test_scaled_kernel_matches_torch_cpu(cuda, src_name, dst_name, scale_name):
    torch = _torch()
    sdt, ddt, scdt = getattr(torch, src_name), getattr(torch, dst_name), getattr(torch, scale_name)
    rng = np.random.default_rng(F8.index(src_name) * 9 + DSTS.index(dst_name) * 3 + ["float32", "bfloat16", "float16"].index(scale_name))
    for R, C, br, bc, n_seg in ((5, 13, 2, 4, 6), (40, 37, 8, 16, 9), (130, 300, 128, 128, 6), (9, 61, 1, 61, 4), (17, 19, 17, 19, 4)):
        src, base, segs, scales, dst_len, where, s, _, (SR, SC) = _rect_case(cuda, rng, sdt, ddt, scdt, R, C, br, bc, n_seg)
        got = _scaled_on_device(cuda, src, segs, scales, dst_len)
        want = np.full(dst_len, GUARD, dtype=np.uint8)
        for at, dp, rows in where:
            for i, v in enumerate(rows):
                idx = torch.from_numpy((v // C // br) * SC + (v % C) // bc)
                ref = _reference(_view(src[base + v], sdt), s, idx, ddt)
                n = v.size * ddt.itemsize
                _assert_same(_view(got[at + i * dp:at + i * dp + n], ddt), ref, (R, C, at, i))
                want[at + i * dp:at + i * dp + n] = got[at + i * dp:at + i * dp + n]
        assert np.array_equal(got, want), "bytes outside the destination rows were written"


def test_mixed_table_scaled_unscaled_fp8_and_plain_cast(cuda):
    """one launch of the scaled instance over scaled, unscaled-FP8 and plain-cast segments: each converts as its own kind"""
    torch = _torch()
    rng = np.random.default_rng(77)
    src = rng.integers(0, 256, size=4096, dtype=np.uint8)
    s = _scales(rng, 4, torch.float32).to(cuda)
    segs = [(3, 0, 1000, 1, 0, 0, _lib.DTYPE_F8_E4M3, _lib.DTYPE_BF16), (1003, 2048, 500, 1, 0, 0, _lib.DTYPE_F8_E5M2, _lib.DTYPE_F32),
            (1504, 4096, 600, 1, 0, 0, _lib.DTYPE_F32, _lib.DTYPE_F16)]
    scales = [(s.data_ptr(), _lib.DTYPE_F32, 1, 250, 4, 1000, 0, 0), None, None]
    got = _scaled_on_device(cuda, src, segs, scales, 4096 + 1200 + 64)
    x = _view(src[3:1003], torch.float8_e4m3fn)
    _assert_same(_view(got[:2000], torch.bfloat16), _reference(x, s.cpu(), torch.arange(1000) // 250, torch.bfloat16))
    _assert_same(_view(got[2048:4048], torch.float32), _view(src[1003:1503], torch.float8_e5m2).to(torch.float32))
    _assert_same(_view(got[4096:5296], torch.float16), _view(src[1504:3904], torch.float32).to(torch.float16))
    assert (got[2000:2048] == GUARD).all() and (got[4048:4096] == GUARD).all() and (got[5296:] == GUARD).all()


# ---- scaled reads through the reader

def _range_sets(n):
    """(file_off, row_len, rows, file_pitch, src dtype, dst dtype, scale) with scale = (dtype, scale_rows, scale_cols, block_rows,
    block_cols, cols, first_elem) or None; FP8 rows are bytes"""
    return [
        # a dim-1 slice of a 40 x 3000 weight with 128 x 128 block scales, next to an unscaled FP8 range and a plain one
        [(7, 1500, 40, 3000, "float8_e4m3fn", "bfloat16", ("float32", 1, 24, 128, 128, 3000, 1000)),
         (121000, 5 * BS + 3, 1, 0, "float8_e5m2", "float32", None), (8 * BS, 2 * BS, 1, 0, "uint8", "uint8", None)],
        # a whole per-row-scaled weight (one long row crossing view rows: cols 2001), a plain cast range, a per-tensor scaled one
        [(3, 50 * 2001, 1, 0, "float8_e5m2", "float16", ("bfloat16", 50, 1, 1, 2001, 2001, 0)),
         (110000, 3 * BS, 1, 0, "float32", "bfloat16", None),
         (310001, 64 * 999, 1, 0, "float8_e4m3fn", "float32", ("float32", 1, 1, 64, 999, 999, 0))],
        # a dim-0 slice of a 300 x 257 weight with 64 x 32 blocks, rows 100..300 (first_elem = 100 * 257), and an empty scaled range
        [(1000 + 100 * 257, 200 * 257, 1, 0, "float8_e4m3fn", "bfloat16", ("float16", 5, 9, 64, 32, 257, 100 * 257)),
         (n - 64, 0, 3, 8, "float8_e4m3fn", "float32", ("float32", 1, 1, 1, 1, 1, 0))],
    ]


def _place(rng, ranges, cuda):
    torch = _torch()
    at, out = 64, []
    for off, L, R, P, s, d, _ in ranges:
        ss, ds = getattr(torch, s).itemsize, getattr(torch, d).itemsize
        at += (-at) % ds + ds * (1 + int(rng.integers(0, 8)))
        drow = L // ss * ds
        dp = drow + (ds * int(rng.integers(1, 5)) if R > 1 else 0)
        out.append((at, dp))
        at += max(0, R - 1) * dp + drow + 16
    return torch.full((at + 64,), GUARD, dtype=torch.uint8, device=cuda), out


def _scale_tensors(rng, ranges, cuda):
    torch = _torch()
    return [None if sc is None else _scales(rng, sc[1] * sc[2], getattr(torch, sc[0])).to(cuda) for *_, sc in ranges]


def _rs(ranges, dst, base, scl):
    torch = _torch()
    out = []
    for (off, L, R, P, s, d, sc), (at, dp), t in zip(ranges, dst, scl):
        scale = None if sc is None else (t.data_ptr(), t.dtype) + tuple(sc[1:])
        out.append((off, L, R, P, base + at, dp, getattr(torch, s), getattr(torch, d), scale))
    return out


def _check_landed(pool, ranges, dst, scl, want):
    torch = _torch()
    host = pool.cpu().numpy().copy()
    for (off, L, R, P, s, d, sc), (at, dp), t in zip(ranges, dst, scl):
        sdt, ddt = getattr(torch, s), getattr(torch, d)
        drow = L // sdt.itemsize * ddt.itemsize
        for k in range(R if L else 0):
            src = _view(want[off + k * P:off + k * P + L], sdt)
            got = host[at + k * dp:at + k * dp + drow]
            if sc is not None:
                _, SR, SC, br, bc, cols, first = sc
                v = first + k * P + np.arange(L)
                ref = _reference(src, t.cpu(), torch.from_numpy((v // cols // br) * SC + (v % cols) // bc), ddt)
                _assert_same(_view(got, ddt), ref, (off, k))
            elif sdt == ddt:
                assert np.array_equal(got, want[off + k * P:off + k * P + L]), (off, k)
            else:
                _assert_same(_view(got, ddt), src.to(ddt), (off, k))
            host[at + k * dp:at + k * dp + drow] = GUARD
    assert (host == GUARD).all(), "bytes outside the destination rows were written"


def _touched(ranges):
    return sorted({b for off, L, R, P, *_ in ranges if L for k in range(R) for b in range((off + k * P) // BS, (off + k * P + L - 1) // BS + 1)})


@pytest.mark.parametrize("copy_group", [1, 4])
@pytest.mark.parametrize("mode", list(MODES))
def test_scaled_reads_dequantize_and_touched_blocks_verify_whole(cuda, cluster, mode, copy_group):
    torch = _torch()
    plain, arena, _ = cluster
    n, ino = 24 * BS, 9950 + 2 * list(MODES).index(mode) + copy_group // 4
    w = arena if mode == "arena" else plain
    path = "/sc/%s%d" % (mode, copy_group)
    man = w.create_file(path, ino, n, BS, threads=2)
    want = np.frombuffer(synth.file_bytes(ino, n, BS), dtype=np.uint8)
    crcs = clib.crc_blocks(1, want, BS).astype(np.uint64)
    rng = np.random.default_rng(19 + copy_group)
    with _fs_for(cluster, mode, man, copy_group) as fs:
        for ranges in _range_sets(n):
            pool, dst = _place(rng, ranges, cuda)
            scl = _scale_tensors(rng, ranges, cuda)
            r = fs.open(path)
            got = r.readv_scaled_device(_rs(ranges, dst, pool.data_ptr(), scl), torch.cuda.current_stream().cuda_stream)
            assert got == sum(L // getattr(torch, s).itemsize * getattr(torch, d).itemsize * R for _, L, R, _, s, d, _ in ranges)
            s, bad, ver = r.verify()
            torch.cuda.synchronize()
            _check_landed(pool, ranges, dst, scl, want)
            touched = _touched(ranges)
            assert bad == 0 and ver == len(touched) and s == int(crcs[touched].sum()), (ver, touched)
            r.complete()


def test_a_corrupt_byte_in_a_dequantized_block_is_counted_and_holes_are_zeros(cuda, cluster):
    torch = _torch()
    plain, _, d = cluster
    n, ino = 8 * BS, 9965
    man = plain.create_file("/sc/bad", ino, n, BS, threads=2) + plain.create_file("/sc/holes", ino + 1, 7 * BS, BS, mode=2, hole_every=3, threads=2)
    _flip(layout.block_path(d + "/mem/curvine", layout.create_block_id(ino, 5)), 4096 * 3 + 100)
    with F.CurvineFileSystem(_conf(True)) as fs:
        fs.load_namespace(man)
        s = torch.full((4,), 0.5, dtype=torch.float32, device=cuda)
        out = torch.empty(4 * BS, dtype=torch.bfloat16, device=cuda)
        r = fs.open("/sc/bad")
        r.readv_scaled_device([(4 * BS, 4 * BS, 1, 0, out.data_ptr(), 0, torch.float8_e4m3fn, torch.bfloat16,
                                (s.data_ptr(), torch.float32, 4, 1, 1, BS, BS, 0))])
        assert r.verify()[1:] == (1, 4)
        r.complete()
        r = fs.open("/sc/holes")  # blocks 2 and 5 are holes
        out.fill_(1.0)
        r.readv_scaled_device([(2 * BS, BS, 1, 0, out.data_ptr(), 0, torch.float8_e5m2, torch.bfloat16, (s.data_ptr(), torch.float32, 1, 1, 1, BS, BS, 0))])
        assert r.verify()[1] == 0
        torch.cuda.synchronize()
        assert not out[:BS].cpu().view(torch.int16).numpy().any()  # zeros times a scale: zeros
        r.complete()


def test_scaled_read_is_ordered_on_the_callers_stream(cuda, cluster):
    torch = _torch()
    from test_zzz_stream_order_gpu import CallerStream
    plain, _, _ = cluster
    n, ino = 12 * BS, 9967
    man = plain.create_file("/sc/so", ino, n, BS, threads=2)
    want = np.frombuffer(synth.file_bytes(ino, n, BS), dtype=np.uint8)
    off, L = 1000, 10 * BS
    cs = None
    try:
        with F.CurvineFileSystem(_conf(False)) as fs:
            fs.load_namespace(man)
            cs = CallerStream(torch)
            scale = torch.zeros(10, dtype=torch.float32, device=cuda)
            sval = torch.from_numpy(np.ldexp(1.0, np.arange(-5, 5)).astype(np.float32)).to(cuda)
            exp = _reference(_view(want[off:off + L], torch.float8_e4m3fn), sval.cpu(), torch.arange(L) // BS, torch.bfloat16)
            dst = torch.zeros(2 * L, dtype=torch.uint8, device=cuda)
            out = torch.zeros(2 * L, dtype=torch.uint8, device=cuda)
            slow = torch.zeros(8 << 20, dtype=torch.uint8, device=cuda)
            torch.cuda.synchronize()
            for rnd in range(2):
                for _ in range(4):
                    cs.fill(slow, rnd)
                for v in (0xE0, 0xE1 + rnd):
                    cs.fill(dst, v)  # pending writes to the destination, enqueued BEFORE the read
                cs.copy(scale.view(torch.uint8), sval.view(torch.uint8))  # and the scales: the read must see them
                r = fs.open("/sc/so")
                rs = [(off, L, 1, 0, dst.data_ptr(), 0, torch.float8_e4m3fn, torch.bfloat16, (scale.data_ptr(), torch.float32, 1, 10, 1, BS, L, 0))]
                assert r.readv_scaled_device(rs, cs.handle) == 2 * L
                cs.copy(out, dst)  # enqueued AFTER the read, same stream, no host synchronisation in between
                cs.synchronize()
                _assert_same(out.cpu().view(torch.bfloat16), exp, "round %d" % rnd)
                assert r.verify()[1] == 0
                r.complete()
                out.zero_()
                scale.zero_()
    finally:
        if cs is not None:
            cs.close()


F32, F16, BF16, E4, E5 = _lib.DTYPE_F32, _lib.DTYPE_F16, _lib.DTYPE_BF16, _lib.DTYPE_F8_E4M3, _lib.DTYPE_F8_E5M2
GOOD = dict(src=E4, dst=BF16, sdt=F32, srows=2, scols=2, br=4, bc=8, cols=16, first=0)


@pytest.mark.parametrize("change,what", [
    (dict(src=F32), "is scaled but its source dtype 1 is not F8"),
    (dict(src=BF16, dst=F32), "is scaled but its source dtype 3"),
    (dict(dst=E5), "F8 is a source type only"),
    (dict(dst=E4, src=E4), "F8 is a source type only"),
    (dict(sdt=E4), "unknown scale dtype code 4"),
    (dict(sdt=0), "unknown scale dtype code 0"),
    (dict(br=0), "must be at least 1"), (dict(bc=0), "must be at least 1"), (dict(cols=0), "must be at least 1"),
    (dict(srows=0), "must be at least 1"), (dict(scols=-1), "must be at least 1"),
    (dict(first=-1), "negative first_elem"),
    (dict(scols=1), "scale_cols 1 < ceil(cols / block_cols) = 2"),
    (dict(first=7 * 16), "maps to scale row 2, but the scale has 2 rows"),  # 32 elements from view row 7: rows 7..8, scale row 2
    (dict(first=(1 << 63) - 10), "overflows int64"),
    (dict(srows=1 << 62, scols=4), "overflows"),
    (dict(scale="host"), "range 1 scale"),
])
def test_scaled_range_errors_name_the_range_and_leave_the_reader_usable(cuda, cluster, change, what):
    torch = _torch()
    if MOCK and change.get("scale"):
        pytest.skip("the host stand-in treats host memory as device memory")
    plain, _, _ = cluster
    n, ino = 4 * BS, 9970
    man = plain.create_file("/sc/err", ino, n, BS, threads=2)
    with F.CurvineFileSystem(_conf(True)) as fs:
        fs.load_namespace(man)
        r = fs.open("/sc/err")
        out = torch.zeros(256, dtype=torch.float32, device=cuda)
        scale = torch.ones(4, dtype=torch.float32, device=cuda)
        host = (ctypes.c_float * 4)()
        c = dict(GOOD, **change)
        arr = (_lib.CvScaledRange * 2)()
        a = arr[0].cast
        a.file_off, a.row_len, a.rows, a.d_dst, a.src_dtype, a.dst_dtype = 0, 16, 1, out.data_ptr(), E4, F32  # fine: the error names range 1
        b, s = arr[1].cast, arr[1]
        b.file_off, b.row_len, b.rows, b.d_dst, b.src_dtype, b.dst_dtype = 100, 32, 1, out.data_ptr() + 512, c["src"], c["dst"]
        s.d_scale = ctypes.addressof(host) if c.get("scale") == "host" else scale.data_ptr()
        s.scale_dtype, s.scale_rows, s.scale_cols, s.block_rows, s.block_cols, s.cols, s.first_elem = (
            c["sdt"], c["srows"], c["scols"], c["br"], c["bc"], c["cols"], c["first"])
        nb = ctypes.c_int64()
        assert _lib.lib().cv_readv_scaled_device(r._h, arr, 2, None, ctypes.byref(nb)) < 0
        msg = _lib.lib().cv_last_error().decode()
        assert "range 1" in msg and what in msg, msg
        # the same reader, the same ranges made right: it dequantizes
        b.src_dtype, b.dst_dtype = E4, BF16
        s.d_scale, s.scale_dtype, s.scale_rows, s.scale_cols, s.block_rows, s.block_cols, s.cols, s.first_elem = (
            scale.data_ptr(), F32, 2, 2, 4, 8, 16, 0)
        assert _lib.lib().cv_readv_scaled_device(r._h, arr, 2, None, ctypes.byref(nb)) == 0 and nb.value == 16 * 4 + 32 * 2
        assert r.verify()[1] == 0
        torch.cuda.synchronize()
        want = np.frombuffer(synth.file_bytes(ino, n, BS), dtype=np.uint8)
        _assert_same(out[128:144].cpu().view(torch.bfloat16)[:32], _view(want[100:132], torch.float8_e4m3fn).to(torch.bfloat16))
        r.complete()


# ---- safetensors.load_file(dtype=..., scales=..., scale_block=...)

def _fp8_checkpoint(torch):
    """FP8 weights with per-tensor, per-row and 128 x 128 block scales (float32 and bfloat16), a weight of another FP8 format, and the
    float and integer tensors around them -> ({name: CPU tensor}, scales, scale_block)"""
    g = torch.Generator().manual_seed(23)

    def fp8(shape, dt):
        return torch.randint(0, 256, shape, generator=g, dtype=torch.int32).to(torch.uint8).view(dt)

    def sc(shape, dt):
        return (torch.rand(shape, generator=g) * 2.0 ** torch.randint(-12, 4, shape, generator=g).float()).to(dt)

    out = {"q_proj.weight": fp8((300, 260), torch.float8_e4m3fn), "q_proj.weight_scale_inv": sc((3, 3), torch.float32),
           "o_proj.weight": fp8((96, 130), torch.float8_e4m3fn), "o_proj.weight_scale": sc((96, 1), torch.bfloat16),
           "gate.weight": fp8((64, 40), torch.float8_e5m2), "gate.weight_scale": sc((1,), torch.float32),
           "norm": torch.randn((77,), generator=g), "ids": torch.randint(0, 1000, (8, 6), generator=g), "odd_scale": sc((), torch.float32),
           "odd": fp8((33,), torch.float8_e4m3fn)}
    scales = {"q_proj.weight": "q_proj.weight_scale_inv", "o_proj.weight": "o_proj.weight_scale", "gate.weight": "gate.weight_scale",
              "odd": "odd_scale"}
    return out, scales, (128, 128)


def _dequant(w, s, block, target):
    """the CPU reference: DeepSeek's formula, (w.float() * s_full.float()).to(target) with s_full the scale grid expanded and cropped"""
    R = w.shape[0] if w.dim() == 2 else 1
    C = w.shape[-1] if w.dim() else 1
    sf = s.float()
    if s.numel() == 1:
        full = sf.reshape(1, 1).expand(R, C)
    elif s.dim() == 2 and s.shape[1] == 1:
        full = sf.expand(R, C)
    else:
        full = sf.repeat_interleave(block[0], 0).repeat_interleave(block[1], 1)[:R, :C]
    return (w.float().reshape(R, C) * full).reshape(w.shape).to(target)


def test_load_file_scales_equals_the_cpu_dequant(cuda, cluster):
    torch = _torch()
    from test_readv_plan import write_safetensors
    from test_zzz_readv_gpu import _bytes
    plain, _, _ = cluster
    dev = "cpu" if MOCK else cuda
    src, scales, block = _fp8_checkpoint(torch)
    names = {dt: name for name, dt in ST.dtypes().items()}
    blob = write_safetensors([(k, names[t.dtype], tuple(t.shape), _bytes(t)) for k, t in src.items()], pad_to=8)
    path = "/sc/model.safetensors"

    def expect(name, target, t=None):
        t = src[name] if t is None else t
        if name in scales:
            return _dequant(t, src[scales[name]], block, target)
        return t.to(target) if t.dtype.is_floating_point else t

    with F.CurvineFileSystem(_conf(True)) as fs:
        wr = fs.create(path, 9975, BS, plain.port, chunk_size=32768)
        wr.write(blob)
        wr.complete()
        for target in (torch.bfloat16, torch.float16, torch.float32):
            got = ST.load_file(fs, path, device=dev, dtype=target, scales=scales, scale_block=block)
            assert set(got) == set(src)
            for name in src:
                want = expect(name, target)
                assert got[name].dtype == want.dtype and tuple(got[name].shape) == tuple(src[name].shape), name
                if want.dtype.is_floating_point:
                    _assert_same(got[name].cpu().reshape(-1), want.reshape(-1), (name, target))
                else:
                    assert _bytes(got[name]) == _bytes(want), name
        for dim in (0, 1):
            for rank in range(2):
                slices = {}
                for name in ("q_proj.weight", "o_proj.weight", "gate.weight", "ids"):
                    size = src[name].shape[dim]
                    slices[name] = (dim, rank * size // 2, (rank + 1) * size // 2)
                got = ST.load_file(fs, path, device=dev, slices=slices, dtype=torch.bfloat16, scales=scales, scale_block=block,
                                   names=list(slices) + ["norm"])
                for name, (d, a, b) in slices.items():
                    exp = expect(name, torch.bfloat16).narrow(d, a, b - a).contiguous()
                    assert tuple(got[name].shape) == tuple(exp.shape), name
                    if exp.dtype.is_floating_point:
                        _assert_same(got[name].cpu().reshape(-1), exp.reshape(-1), (name, dim, rank))
                    else:
                        assert _bytes(got[name]) == _bytes(exp), name
        from curvine_b200 import curvinefs
        client = curvinefs.CurvineClient.__new__(curvinefs.CurvineClient)
        client.file_system_ptr = fs
        via = client.load_safetensors(path, device=dev, names=["o_proj.weight"], dtype=torch.float32, scales=scales, scale_block=block)
        _assert_same(via["o_proj.weight"].cpu().reshape(-1), expect("o_proj.weight", torch.float32).reshape(-1))
        client.file_system_ptr = None


# ---- the scale walk reads no scale past the caller's buffer

class _GuardedScales:
    """host memory whose last bytes sit right in front of a PROT_NONE page: a read one element past the scales faults.  Only on the
    host-side stand-ins, where the kernels run on host cores and "device memory" is host memory."""

    def __init__(self, values):
        import mmap
        self.page = mmap.PAGESIZE
        raw = values.contiguous().view(_torch().uint8).numpy().tobytes()
        assert len(raw) <= self.page
        self.m = mmap.mmap(-1, 2 * self.page, prot=mmap.PROT_READ | mmap.PROT_WRITE)
        self.anchor = ctypes.c_char.from_buffer(self.m)
        base = ctypes.addressof(self.anchor)
        self.libc = ctypes.CDLL(None, use_errno=True)
        assert self.libc.mprotect(ctypes.c_void_p(base + self.page), ctypes.c_size_t(self.page), 0) == 0
        self.ptr = base + self.page - len(raw)
        ctypes.memmove(self.ptr, raw, len(raw))
        self.base = base

    def close(self):
        self.libc.mprotect(ctypes.c_void_p(self.base + self.page), ctypes.c_size_t(self.page), 3)
        del self.anchor
        self.m.close()


# (rows, cols, block_rows, block_cols, scale grid): per tensor, per row, and tiles whose grid ends exactly at the weight's last row
WALK_CASES = [(7, 13, 7, 13, (1, 1)), (9, 61, 1, 61, (9, 1)), (256, 40, 128, 16, (2, 3)), (6, 40, 3, 8, (2, 5))]


@pytest.mark.parametrize("R,C,br,bc,grid", WALK_CASES)
def test_the_scale_walk_stays_inside_the_scale_buffer(cuda, R, C, br, bc, grid):
    """The last element of the weight, in a partial last chunk and in a whole last chunk that crosses a view row, for every
    destination alignment: the scale walk reads the last scale, never the one past it."""
    if not MOCK:
        pytest.skip("needs a guard page behind the scales: on the GPU a stray read would only show as a fault")
    torch = _torch()
    rng = np.random.default_rng(R * C)
    SR, SC = grid
    s = _scales(rng, SR * SC, torch.float32)
    g = _GuardedScales(s)
    try:
        src = rng.integers(0, 256, size=R * C + 16, dtype=np.uint8)
        segs, scales, where, at = [], [], [], 0
        for shift in range(8):  # destination offsets 0..7 bf16 elements past a 16-byte boundary: every place the last chunk can end
            for first in (0, R * C - 8 - shift, R * C - 1):
                n = R * C - first
                if n <= 0:
                    continue
                at += (-at) % 16 + 2 * shift
                segs.append((first, at, n, 1, 0, 0, _lib.DTYPE_F8_E4M3, _lib.DTYPE_BF16))
                scales.append((g.ptr, _lib.DTYPE_F32, br, bc, SC, C, first, 0))
                where.append((at, first, n))
                at += 2 * n + 16
        got = _scaled_on_device(cuda, src, segs, scales, at + 64)
        for at, first, n in where:
            v = np.arange(first, first + n)
            idx = torch.from_numpy((v // C // br) * SC + (v % C) // bc)
            _assert_same(_view(got[at:at + 2 * n], torch.bfloat16), _reference(_view(src[v], torch.float8_e4m3fn), s, idx, torch.bfloat16),
                         (first, at))
    finally:
        g.close()


def test_a_scaled_read_to_the_weights_end_stays_inside_the_scale_buffer(cuda, cluster):
    """the same through cv_readv_scaled_device: a per-tensor scaled weight that ends the file, its one scale in front of the guard page"""
    if not MOCK:
        pytest.skip("needs a guard page behind the scales: on the GPU a stray read would only show as a fault")
    torch = _torch()
    plain, _, _ = cluster
    n, ino = 3 * BS + 77, 9978
    man = plain.create_file("/sc/end", ino, n, BS, threads=2)
    want = np.frombuffer(synth.file_bytes(ino, n, BS), dtype=np.uint8)
    s = torch.tensor([0.375], dtype=torch.float32)
    g = _GuardedScales(s)
    try:
        with F.CurvineFileSystem(_conf(True)) as fs:
            fs.load_namespace(man)
            r = fs.open("/sc/end")
            L = n - 1001
            out = torch.zeros(L + 3, dtype=torch.bfloat16, device=cuda)
            for k in range(3):  # three destination alignments of the weight's last chunk
                r.readv_scaled_device([(1001, L, 1, 0, out.data_ptr() + 2 * k, 0, torch.float8_e5m2, torch.bfloat16,
                                        (g.ptr, torch.float32, 1, 1, 1, L, L, 0))])
                assert r.verify()[1] == 0
                torch.cuda.synchronize()
                ref = _reference(_view(want[1001:], torch.float8_e5m2), s, torch.zeros(L, dtype=torch.int64), torch.bfloat16)
                _assert_same(out[k:k + L].cpu(), ref, k)
            r.complete()
    finally:
        g.close()
