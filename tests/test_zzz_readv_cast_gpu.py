"""Cast on load on the GPU: the conversion kernel (cvk_gather_cast) bit-exact against torch's CPU Tensor.to() for all six conversions
between float32, float16 and bfloat16, cast reads through the reader (cv_readv_cast_device) in every read mode, and
safetensors.load_file(dtype=...) against load_file() followed by .to() on the CPU.  Runs on the host-side stand-ins too
(tests/simt_emu), where "device memory" is host memory."""
import os
import shutil
import tempfile

import numpy as np
import pytest

from curvine_b200 import _lib
from curvine_b200 import fs as F
from curvine_b200 import safetensors as ST
from oracle import clib, layout, synth

pytestmark = pytest.mark.gpu
MOCK = bool(os.environ.get("CV_TEST_MOCK_CUDA_LIB"))
BS = 64 << 10
GUARD = 0x5A


def _torch():
    import torch
    return torch


def _code(dt):
    torch = _torch()
    return {torch.float32: _lib.DTYPE_F32, torch.float16: _lib.DTYPE_F16, torch.bfloat16: _lib.DTYPE_BF16}[dt]


def _int_view(dt):
    torch = _torch()
    return torch.int32 if dt.itemsize == 4 else torch.int16


def _assert_cast_equal(got, src, ddt, what=""):
    """got (ddt tensor) == src.to(ddt) on the CPU bit for bit, except that a NaN only has to stay a NaN"""
    torch = _torch()
    want = src.to(ddt)
    nan = torch.isnan(src.float())
    gi, wi = got.view(_int_view(ddt)), want.view(_int_view(ddt))
    bad = (gi != wi) & ~nan
    assert not bool(bad.any()), (what, src[bad][:8], got[bad][:8], want[bad][:8])
    assert bool(torch.isnan(got.float()[nan]).all()), what


def _cast_on_device(cuda, src_bytes, segs, dst_len):
    """run cvk_gather_cast over uint8 `src_bytes` with `segs` into a guard-filled buffer of dst_len bytes -> its bytes (numpy)"""
    torch = _torch()
    from curvine_b200 import kernels as K
    d_src = torch.from_numpy(np.ascontiguousarray(src_bytes)).to(cuda)
    dst = torch.full((dst_len,), GUARD, dtype=torch.uint8, device=cuda)
    d_segs, total = K.cast_segs_to_device(segs, cuda) if segs else (None, 0)
    K.gather_cast(d_src, d_segs, len(segs), total, dst)
    torch.cuda.synchronize()
    return dst.cpu().numpy()


def _view(raw, dt):
    torch = _torch()
    return torch.from_numpy(np.array(raw, dtype=np.uint8)).view(dt)


FLOATS = ["float32", "float16", "bfloat16"]
PAIRS = [(a, b) for a in FLOATS for b in FLOATS if a != b]


# ---- cvk_gather_cast against torch CPU .to()

def _f32_cases():
    """bit patterns of float32 sources: the edges of every conversion, then a seeded random sample"""
    special = [0, 0x80000000, 0x7F800000, 0xFF800000, 0x7F7FFFFF, 0xFF7FFFFF, 0x00000001, 0x807FFFFF, 0x00800000, 0x7FC00000, 0xFFC00001,
               0x7F800001]
    for e in range(0x66, 0x72):  # around the float16 subnormal range, 2^-25 .. 2^-14
        for m in (0, 1, 0x1FFF, 0x2000, 0x3FFFFF, 0x400000, 0x400001, 0x7FFFFF):
            special += [(e << 23) | m, 0x80000000 | (e << 23) | m]
    for base in (0x477FE000, 0x477FF000, 0x477FEFFF, 0x477FF001, 0x47800000, 0x38800000, 0x387FF000, 0x33000000, 0x33000001):
        special += [base - 1, base, base + 1]  # largest finite float16, the overflow edge, the normal/subnormal edge, 2^-25
    for hi in (0x3F80, 0x3F81, 0x7F7F, 0x0001, 0x0080):  # bfloat16 ties: the dropped half exactly 0x8000, below and above it
        for lo in (0x7FFF, 0x8000, 0x8001, 0x0000, 0xFFFF):
            special.append((hi << 16) | lo)
    for h in (0x3C00, 0x3C01, 0x0001, 0x03FF, 0x7BFF):  # float16 ties: the 13 dropped bits exactly 0x1000
        f = int(np.array([h], dtype=np.uint16).view(np.float16).astype(np.float32).view(np.uint32)[0])
        special += [f + 0x1000, f + 0xFFF, f + 0x1001, f + 0x3000]
    rnd = np.random.default_rng(5).integers(0, 1 << 32, size=1 << 16, dtype=np.uint64).astype(np.uint32)
    return np.concatenate([np.array(special, dtype=np.uint64).astype(np.uint32), rnd])


@pytest.mark.parametrize("src_name,dst_name", PAIRS)
def test_cast_kernel_is_bit_exact_against_torch_cpu(cuda, src_name, dst_name):
    """every one of the 65,536 bit patterns of a 16-bit source; float32 edges and a random sample of bit patterns"""
    torch = _torch()
    sdt, ddt = getattr(torch, src_name), getattr(torch, dst_name)
    if sdt.itemsize == 2:
        raw = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.uint8)
    else:
        raw = _f32_cases().view(np.uint8)
    n = raw.size // sdt.itemsize
    got = _cast_on_device(cuda, raw, [(0, 0, n, 1, 0, 0, _code(sdt), _code(ddt))], n * ddt.itemsize)
    _assert_cast_equal(_view(got, ddt), _view(raw, sdt), ddt, (src_name, dst_name))


def _layout_case(rng, sdt, ddt, n_seg, max_rows, max_elems):
    """segments at element-only alignment: source and destination offsets anywhere their element size allows, multi-row segments with
    pitches, guard bytes between destination rows, zero-length segments -> (src bytes, segs, dst_len)"""
    ss, ds = sdt.itemsize, ddt.itemsize
    segs, at_src, at_dst = [], 16, 16
    for k in range(n_seg):
        elems = int(rng.integers(1, max_elems + 1))
        rows = int(rng.integers(1, max_rows + 1))
        if k % 5 == 4:
            elems, rows = (0, rows) if k % 2 else (elems, 0)
        sp = elems * ss + ss * int(rng.integers(0, 9))
        dp = elems * ds + ds * int(rng.integers(1, 9))
        so = at_src + ss * int(rng.integers(0, 16 // ss + 1))
        do = at_dst + ds * int(rng.integers(0, 16 // ds + 1))
        segs.append((so, do, elems, rows, sp, dp, _code(sdt), _code(ddt)))
        at_src = so + max(rows, 1) * sp + 16
        at_dst = do + max(rows, 1) * dp + 16
    src = np.random.default_rng(int(rng.integers(1 << 30))).integers(0, 256, size=at_src + 64, dtype=np.uint8)
    return src, segs, at_dst + 64


def _expect_layout(src, segs, dst_len, sdt, ddt):
    torch = _torch()
    want = np.full(dst_len, GUARD, dtype=np.uint8)
    for so, do, elems, rows, sp, dp, _, _ in segs:
        for k in range(rows if elems else 0):
            row = _view(src[so + k * sp:so + k * sp + elems * sdt.itemsize], sdt)
            out = row.to(ddt).view(torch.uint8).numpy()
            want[do + k * dp:do + k * dp + out.size] = out
    return want


def _check_rows(got, src, segs, dst_len, sdt, ddt):
    """every row of every segment converted (NaN payloads may differ), every byte outside the rows untouched"""
    want = _expect_layout(src, segs, dst_len, sdt, ddt)
    for so, do, elems, rows, sp, dp, _, _ in segs:
        for k in range(rows if elems else 0):
            s = _view(src[so + k * sp:so + k * sp + elems * sdt.itemsize], sdt)
            _assert_cast_equal(_view(got[do + k * dp:do + k * dp + elems * ddt.itemsize], ddt), s, ddt, (so, k))
            want[do + k * dp:do + k * dp + elems * ddt.itemsize] = got[do + k * dp:do + k * dp + elems * ddt.itemsize]
    assert np.array_equal(got, want), "bytes outside the destination rows were written"


@pytest.mark.parametrize("src_name,dst_name", PAIRS)
def test_cast_kernel_rows_pitches_alignment_and_guards(cuda, src_name, dst_name):
    torch = _torch()
    sdt, ddt = getattr(torch, src_name), getattr(torch, dst_name)
    rng = np.random.default_rng(17 + FLOATS.index(src_name) * 3 + FLOATS.index(dst_name))
    for n_seg, max_rows, max_elems in ((1, 1, 3), (1, 40, 37), (9, 12, 70), (25, 3, 300)):
        src, segs, dst_len = _layout_case(rng, sdt, ddt, n_seg, max_rows, max_elems)
        _check_rows(_cast_on_device(cuda, src, segs, dst_len), src, segs, dst_len, sdt, ddt)


def test_cast_kernel_spreads_many_short_rows_and_one_long_row(cuda):
    """2^12 rows of 8 elements and one row of 2^17 elements in one table: every element lands, nothing else is touched"""
    torch = _torch()
    rows, long_n = (1 << 12), (1 << 17) + 5
    src = np.random.default_rng(3).integers(0, 256, size=4 * (rows * 8 + long_n) + 64, dtype=np.uint8)
    segs = [(4, 2, 8, rows, 32, 18, _lib.DTYPE_F32, _lib.DTYPE_BF16),
            (4 + 4 * rows * 8 + 4, 2 + 18 * rows + 6, long_n, 1, 0, 0, _lib.DTYPE_F32, _lib.DTYPE_BF16),
            (0, 0, 0, 5, 4, 4, _lib.DTYPE_F32, _lib.DTYPE_BF16)]
    dst_len = 2 + 18 * rows + 6 + 2 * long_n + 32
    _check_rows(_cast_on_device(cuda, src, segs, dst_len), src, segs, dst_len, torch.float32, torch.bfloat16)


# ---- cast reads through the reader

def _conf(sc, copy_group=1, zero_copy=False, arena_dir=None):
    # 8 ring slots: at most 8 boundary blocks are staged per round, so the range sets below take several rounds
    b200 = 'fetch_threads = 2\nverify_batch = 2\npinned_slots = 8\ncopy_group = %d\ngpu_chunk_size = "32KB"\nzero_copy = %s\n' % (
        copy_group, "true" if zero_copy else "false")
    if arena_dir:
        b200 += 'register_threads = 2\narena_register_slice = "4MB"\narena_preregister = ["%s"]\n' % arena_dir
    return F.client_conf(short_circuit=sc, b200=b200)


@pytest.fixture(scope="module")
def cluster():
    d = tempfile.mkdtemp(prefix="cvca", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    plain = F.MiniWorker(["[MEM]" + d + "/mem"])
    arena = F.MiniWorker(["[MEM:16MB]" + d + "/arena"], extra_worker='mem_arena = true\narena_segment = "8MB"\n')
    yield plain, arena, d
    plain.stop()
    arena.stop()
    shutil.rmtree(d, ignore_errors=True)


MODES = {"files": dict(sc=True), "framed": dict(sc=False), "arena": dict(sc=True, zero_copy=True)}


def _fs_for(cluster, mode, man, copy_group):
    plain, arena, d = cluster
    fs = F.CurvineFileSystem(_conf(copy_group=copy_group, arena_dir=d + "/arena" if mode == "arena" else None, **MODES[mode]))
    fs.load_namespace(man)
    if mode == "arena":
        fs.preregister()
        fs.wait_registered()
    return fs


def _range_sets(n):
    """(file_off, row_len, rows, file_pitch, src dtype name, dst dtype name); row_len and the pitches in source bytes"""
    return [
        [(4, n - 8, 1, 0, "float32", "bfloat16")],                                  # the whole file but 8 bytes: every block a boundary block
        [(5000, 3000, (n - 8000) // 12000 + 1, 12000, "bfloat16", "float32")],      # a column: rows across block edges, 2x wider in HBM
        [(100, 2 * BS + 300, 4, 3 * BS + 8, "float16", "bfloat16"), (13 * BS, BS, 1, 0, "uint8", "uint8"),
         (15 * BS + 2, 998, 7, 1000, "bfloat16", "float16")],                      # long rows; a plain whole block; narrow rows
        [(16, 96, 3, 7 * BS + 4, "float32", "float16"), (n - 64, 64, 1, 0, "float16", "float32"), (8, 0, 4, 12, "float32", "bfloat16")],
    ]


def _place(rng, ranges, cuda):
    """destinations at element-aligned odd-ish offsets with guard bytes around and between rows -> (pool, [(dst offset, dst_pitch)])"""
    torch = _torch()
    at, out = 64, []
    for off, L, R, P, s, d in ranges:
        ss, ds = getattr(torch, s).itemsize, getattr(torch, d).itemsize
        at += (-at) % ds + ds * (1 + int(rng.integers(0, 8)))
        drow = L // ss * ds
        dp = drow + (ds * int(rng.integers(1, 5)) if R > 1 else 0)
        out.append((at, dp))
        at += max(0, R - 1) * dp + drow + 16
    return torch.full((at + 64,), GUARD, dtype=torch.uint8, device=cuda), out


def _check_landed(pool, ranges, dst, want):
    torch = _torch()
    host = pool.cpu().numpy().copy()
    for (off, L, R, P, s, d), (at, dp) in zip(ranges, dst):
        sdt, ddt = getattr(torch, s), getattr(torch, d)
        drow = L // sdt.itemsize * ddt.itemsize
        for k in range(R if L else 0):
            src = want[off + k * P:off + k * P + L]
            got = host[at + k * dp:at + k * dp + drow]
            if sdt == ddt:
                assert np.array_equal(got, src), (off, k)
            else:
                _assert_cast_equal(_view(got, ddt), _view(src, sdt), ddt, (off, k))
            host[at + k * dp:at + k * dp + drow] = GUARD
    assert (host == GUARD).all(), "bytes outside the destination rows were written"


def _touched(ranges):
    return sorted({b for off, L, R, P, _, _ in ranges if L for k in range(R) for b in range((off + k * P) // BS, (off + k * P + L - 1) // BS + 1)})


def _rs(ranges, dst, base):
    torch = _torch()
    return [(off, L, R, P, base + at, dp, getattr(torch, s), getattr(torch, d)) for (off, L, R, P, s, d), (at, dp) in zip(ranges, dst)]


@pytest.mark.parametrize("copy_group", [1, 4])
@pytest.mark.parametrize("mode", list(MODES))
def test_cast_reads_land_converted_and_touched_blocks_verify_whole(cuda, cluster, mode, copy_group):
    torch = _torch()
    plain, arena, _ = cluster
    n, ino = 24 * BS, 9910 + 2 * list(MODES).index(mode) + copy_group // 4
    w = arena if mode == "arena" else plain
    man = w.create_file("/ca/%s%d" % (mode, copy_group), ino, n, BS, threads=2)
    want = np.frombuffer(synth.file_bytes(ino, n, BS), dtype=np.uint8)
    crcs = clib.crc_blocks(1, want, BS).astype(np.uint64)
    rng = np.random.default_rng(9 + copy_group)
    with _fs_for(cluster, mode, man, copy_group) as fs:
        for ranges in _range_sets(n):
            pool, dst = _place(rng, ranges, cuda)
            r = fs.open("/ca/%s%d" % (mode, copy_group))
            r.seek(321)
            rs = _rs(ranges, dst, pool.data_ptr())
            got = r.readv_cast_device(rs, torch.cuda.current_stream().cuda_stream)
            assert got == sum(L // getattr(torch, s).itemsize * getattr(torch, d).itemsize * R for _, L, R, _, s, d in ranges)
            assert r.pos() == 321
            s, bad, ver = r.verify()
            torch.cuda.synchronize()
            _check_landed(pool, ranges, dst, want)
            touched = _touched(ranges)
            assert bad == 0 and ver == len(touched), (ver, touched)
            assert s == int(crcs[touched].sum())
            spans, nb, fetch = r.readv_cast_plan(rs)
            assert nb == len(touched) and fetch == len(touched) * BS
            cast_blocks = {sp[0] for sp in spans if ranges[sp[4]][4] != ranges[sp[4]][5]}
            assert not any(sp[5] for sp in spans if sp[0] in cast_blocks)  # no block a conversion touches is direct
            r.complete()


def test_a_mixed_call_keeps_the_plain_ranges_direct_blocks_direct(cuda, cluster):
    torch = _torch()
    plain, _, _ = cluster
    n, ino = 12 * BS, 9920
    man = plain.create_file("/ca/mixed", ino, n, BS, threads=2)
    want = np.frombuffer(synth.file_bytes(ino, n, BS), dtype=np.uint8)
    ranges = [(0, 3 * BS, 1, 0, "uint8", "uint8"), (3 * BS + 4, 2 * BS, 1, 0, "float32", "bfloat16"), (6 * BS, 4 * BS, 1, 0, "float16", "float16"),
              (10 * BS + 6, 1000, 2, 2000, "bfloat16", "float32")]
    with F.CurvineFileSystem(_conf(True)) as fs:
        fs.load_namespace(man)
        pool, dst = _place(np.random.default_rng(4), ranges, cuda)
        r = fs.open("/ca/mixed")
        rs = _rs(ranges, dst, pool.data_ptr())
        spans, nb, _ = r.readv_cast_plan(rs)
        direct = sorted(sp[0] for sp in spans if sp[5])
        assert direct == [0, 1, 2, 6, 7, 8, 9], direct  # the plain and same-dtype ranges' whole blocks; none of the converting ones
        r.readv_cast_device(rs)
        s, bad, ver = r.verify()
        torch.cuda.synchronize()
        _check_landed(pool, ranges, dst, want)
        assert bad == 0 and ver == len(_touched(ranges))
        r.complete()


def _flip(path, off):
    with open(path, "r+b") as f:
        f.seek(off)
        b = f.read(1)
        f.seek(off)
        f.write(bytes([b[0] ^ 0x20]))


@pytest.mark.parametrize("sc", [True, False])
def test_a_corrupt_byte_in_a_converted_block_is_counted(cuda, cluster, sc):
    torch = _torch()
    plain, _, d = cluster
    n, ino = 8 * BS, 9925 + int(sc)
    man = plain.create_file("/ca/bad%d" % sc, ino, n, BS, threads=2)
    _flip(layout.block_path(d + "/mem/curvine", layout.create_block_id(ino, 5)), 4096 * 3 + 100)
    with F.CurvineFileSystem(_conf(sc)) as fs:
        fs.load_namespace(man)
        out = torch.empty(BS, dtype=torch.bfloat16, device=cuda)  # 4 blocks of float32
        r = fs.open("/ca/bad%d" % sc)
        r.readv_cast_device([(4 * BS, 4 * BS, 1, 0, out.data_ptr(), 0, torch.float32, torch.bfloat16)])
        assert r.verify()[1:] == (1, 4)
        r.complete()


def test_cast_rows_over_hole_blocks_are_zeros(cuda, cluster):
    torch = _torch()
    plain, _, _ = cluster
    n, ino = 7 * BS, 9928
    man = plain.create_file("/ca/holes", ino, n, BS, mode=2, hole_every=3, threads=2)  # blocks 2 and 5 are holes
    want = np.frombuffer(synth.file_bytes(ino, n, BS), dtype=np.uint8).copy()
    for b in (2, 5):
        want[b * BS:(b + 1) * BS] = 0
    ranges = [(BS + 8, 5000, 9, 20000, "float32", "bfloat16"), (5 * BS + 2, BS - 4, 1, 0, "bfloat16", "float32")]
    with F.CurvineFileSystem(_conf(True)) as fs:
        fs.load_namespace(man)
        r = fs.open("/ca/holes")
        pool, dst = _place(np.random.default_rng(2), ranges, cuda)
        r.readv_cast_device(_rs(ranges, dst, pool.data_ptr()))
        s, bad, ver = r.verify()
        torch.cuda.synchronize()
        _check_landed(pool, ranges, dst, want)
        at, _ = dst[1]
        assert not pool[at:at + (BS - 4) * 2].cpu().numpy().any()  # the hole's zeros convert to zeros
        touched = _touched(ranges)
        assert 2 in touched and bad == 0 and ver == len([b for b in touched if b not in (2, 5)])
        r.complete()


def test_cast_read_is_ordered_on_the_callers_stream(cuda, cluster):
    torch = _torch()
    from test_zzz_stream_order_gpu import CallerStream
    plain, _, _ = cluster
    n, ino = 12 * BS, 9929
    man = plain.create_file("/ca/so", ino, n, BS, threads=2)
    want = np.frombuffer(synth.file_bytes(ino, n, BS), dtype=np.uint8)
    off, L = 1000, 10 * BS
    exp = _view(want[off:off + L], torch.float32).to(torch.bfloat16)
    cs = None
    try:
        with F.CurvineFileSystem(_conf(False)) as fs:
            fs.load_namespace(man)
            cs = CallerStream(torch)
            dst = torch.zeros(L // 2, dtype=torch.uint8, device=cuda)
            out = torch.zeros(L // 2, dtype=torch.uint8, device=cuda)
            slow = torch.zeros(8 << 20, dtype=torch.uint8, device=cuda)
            torch.cuda.synchronize()
            for rnd in range(2):
                for _ in range(4):
                    cs.fill(slow, rnd)
                for v in (0xE0, 0xE1 + rnd):
                    cs.fill(dst, v)  # pending writes to the destination, enqueued BEFORE the read
                r = fs.open("/ca/so")
                assert r.readv_cast_device([(off, L, 1, 0, dst.data_ptr(), 0, torch.float32, torch.bfloat16)], cs.handle) == L // 2
                cs.copy(out, dst)  # enqueued AFTER the read, same stream, no host synchronisation in between
                cs.synchronize()
                _assert_cast_equal(out.cpu().view(torch.bfloat16), exp, torch.bfloat16, "round %d" % rnd)
                assert r.verify()[1] == 0
                r.complete()
                out.zero_()
    finally:
        if cs is not None:
            cs.close()


# ---- safetensors.load_file(dtype=...)

def _checkpoint(torch):
    g = torch.Generator().manual_seed(21)
    specs = [("embed", torch.float32, (96, 130)), ("norm", torch.float32, (77,)), ("qkv", torch.float32, (3, 40, 257)),
             ("half", torch.float16, (33, 70)), ("brain", torch.bfloat16, (50, 9)), ("ids", torch.int64, (8, 6)), ("mask", torch.bool, (12, 5, 2)),
             ("empty", torch.float32, (0, 12)), ("big", torch.float32, (40, BS // 16 + 3))]
    out = {}
    for name, dt, shape in specs:
        if dt.is_floating_point:
            t = torch.randn(shape, generator=g, dtype=torch.float32) * 300
            out[name] = t.to(dt)
        else:
            out[name] = torch.randint(0, 2 if dt == torch.bool else 1000, shape, generator=g).to(dt)
    return out


def test_load_file_dtype_equals_cpu_to(cuda, cluster):
    torch = _torch()
    from test_readv_plan import write_safetensors
    from test_zzz_readv_gpu import _bytes
    plain, _, _ = cluster
    dev = "cpu" if MOCK else cuda
    src = _checkpoint(torch)
    names = {dt: name for name, dt in ST.dtypes().items()}
    blob = write_safetensors([(k, names[t.dtype], tuple(t.shape), _bytes(t)) for k, t in src.items()], pad_to=8)
    path = "/ca/model.safetensors"
    with F.CurvineFileSystem(_conf(True)) as fs:
        wr = fs.create(path, 9930, BS, plain.port, chunk_size=32768)
        wr.write(blob)
        wr.complete()
        for target in (torch.bfloat16, torch.float16, torch.float32):
            got = ST.load_file(fs, path, device=dev, dtype=target)
            for name, t in src.items():
                want = t.to(target) if t.dtype.is_floating_point else t
                assert got[name].dtype == want.dtype and tuple(got[name].shape) == tuple(t.shape), name
                assert _bytes(got[name]) == _bytes(want), (name, target)
        sub = ST.load_file(fs, path, device=dev, names=["qkv", "ids"], dtype=torch.bfloat16)
        assert set(sub) == {"qkv", "ids"} and _bytes(sub["qkv"]) == _bytes(src["qkv"].to(torch.bfloat16)) and _bytes(sub["ids"]) == _bytes(src["ids"])
        for dim in (0, 1):
            for rank in range(2):
                slices = {}
                for name, t in src.items():
                    if t.dim() > dim:
                        size = t.shape[dim]
                        slices[name] = (dim, rank * size // 2, (rank + 1) * size // 2)
                got = ST.load_file(fs, path, device=dev, slices=slices, dtype=torch.bfloat16)
                for name, t in src.items():
                    exp = t.narrow(*slices[name][:2], slices[name][2] - slices[name][1]) if name in slices else t
                    exp = exp.contiguous().to(torch.bfloat16) if t.dtype.is_floating_point else exp.contiguous()
                    assert got[name].is_contiguous() and tuple(got[name].shape) == tuple(exp.shape), (name, dim)
                    assert _bytes(got[name]) == _bytes(exp), (name, dim, rank)
        from curvine_b200 import curvinefs
        client = curvinefs.CurvineClient.__new__(curvinefs.CurvineClient)
        client.file_system_ptr = fs
        via = client.load_safetensors(path, device=dev, names=["half"], dtype=torch.float32)
        assert _bytes(via["half"]) == _bytes(src["half"].to(torch.float32))
        client.file_system_ptr = None
