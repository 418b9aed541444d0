"""The launch configurations that small inputs never produce, against the oracle, numpy or torch on the CPU, bit for bit.

  * Every row-walker launcher (K1 crc_blocks, K2 unpack_frames, K4 pack_frames, K3 gather_pages / gather_strided /
    deinterleave_blocks / gather_shards_p2p) at every segment size cvk_tune(4, s) can force, s = 12..20 (units of 4 KiB .. 1 MiB),
    with pieces just below, at and just above 2^s; then one mixed input per launcher that must give the same bytes and CRCs at all
    nine settings, which is what cvk_tune promises.  The suite's other inputs only reach s = 12..15.
  * K1 with total_bytes passed as an upper bound (the header allows it: only the workspace grows), chosen so that the size-derived
    choice lands on each of s = 14..20 -- among them the benchmark's own call, 4 MiB blocks with a 16 GiB bound, at s = 18.
  * K5's scaled instance, directly and through cv_readv_scaled_device, with view positions, view widths and row steps past 2^32:
    the scale walk then takes its 64-bit divisions.

Destinations are guard-filled and the bytes outside what a launcher writes must stay untouched.  Every buffer a walker reads has
SLACK bytes behind it: the walkers may read the rest of a 16-byte granule.  Runs on the host-side stand-ins too (tests/simt_emu);
tests/test_launch_shapes_mutants.py checks there that planted bugs in the walker and in the scale walk make these tests fail."""
import os

import numpy as np
import pytest

from curvine_b200 import _lib
from oracle import clib, synth, wire as W
from test_kernels_gpu import _build_wire, _rand, _to_dev
from test_zzz_readv_cast_gpu import BS, GUARD, MOCK, _fs_for, cluster  # noqa: F401  (cluster: a fixture)
from test_zzz_readv_scaled_gpu import (DSTS, F8, _GuardedScales, _assert_same, _check_landed, _code, _place, _reference, _rs, _scale_tensors,
                                       _scaled_on_device, _scales, _touched, _view)

pytestmark = pytest.mark.gpu

SHIFTS = list(range(12, 21))
SLACK = 64


def _torch():
    import torch
    return torch


def _K():
    from curvine_b200 import kernels as K
    return K


@pytest.fixture
def tune(cuda):
    """cvk_tune(what, value), with the library's defaults -- sizes chosen from the input, small-input kernels on, the default strided
    train -- restored however the test ends"""
    L = _lib.lib()
    try:
        yield lambda what, value: _lib.check(L.cvk_tune(what, value), "cvk_tune(%d, %d)" % (what, value))
    finally:
        for what, value in ((4, 0), (5, 1), (6, 0)):
            L.cvk_tune(what, value)


@pytest.fixture
def seg(request, tune):
    """segment size 2^s forced for every launcher, and the launch train rather than the small-input kernels"""
    tune(4, request.param)
    tune(5, 0)
    return request.param


def _seg_param():
    return pytest.mark.parametrize("seg", SHIFTS, indirect=True, ids=["s%d" % s for s in SHIFTS])


def _guarded(n):
    torch = _torch()
    return torch.full((n,), GUARD, dtype=torch.uint8)


def _dev(a, cuda):
    """numpy bytes on the device with SLACK bytes behind them"""
    return _to_dev(np.concatenate([a, np.zeros(SLACK, dtype=np.uint8)]), cuda)


# ---- one checker per launcher: it runs the launcher, asserts the oracle's result, and returns what it produced


def _check_k1(cuda, lens, poly, seed):
    """K1 over pieces of `lens` (each at another source phase) at base misalignments 0, 1, 7 and 13 -> the CRCs"""
    K = _K()
    offs, pos = [], 0
    for n in lens:
        offs.append(pos)
        pos += n + 5
    data = _rand(pos + 13, seed)
    d = _dev(data, cuda)
    out = []
    for mis in (0, 1, 7, 13):
        got = K.u32(K.crc_blocks(d, offs, lens, poly, base_offset=mis)).tolist()
        want = [clib.crc(poly, data[mis + o:mis + o + n]) for o, n in zip(offs, lens)]
        assert got == want, [(n, mis, hex(g), hex(w)) for n, g, w in zip(lens, got, want) if g != w]
        out += got
    return out


def _check_frames(cuda, blens, chunk, poly, seed):
    """K2 into destinations at misalignments 0 and 5, and K4 back to the wire: bytes, block CRCs, zero error flags, the oracle's wire
    image, and nothing written outside -> (K2 CRCs, K4 CRCs)"""
    torch, K = _torch(), _K()
    blocks = [_rand(n, seed + i) for i, n in enumerate(blens)]
    wire, descs, _, total = _build_wire(blocks, chunk, [seed * 64 + i for i in range(len(blocks))], poly)
    want = np.concatenate(blocks)
    want_crc = [clib.crc(poly, b) for b in blocks]
    d_desc = K.frame_descs_to_device(descs, cuda)
    d_wire = _dev(wire, cuda)
    for mis in (0, 5):
        dst = _guarded(total + mis + SLACK).to(cuda)
        crc, err = K.unpack_frames(d_wire, d_desc, len(descs), len(blocks), dst[mis:], poly, total)
        out = dst.cpu().numpy()
        assert np.array_equal(out[mis:mis + total], want), (blens, chunk, mis)
        assert (out[:mis] == GUARD).all() and (out[mis + total:] == GUARD).all(), (blens, chunk, mis)
        assert K.u32(crc).tolist() == want_crc and (K.u32(err) == 0).all(), (blens, chunk, mis)
    got_wire = _guarded(len(wire) + SLACK).to(cuda)
    crc4 = K.u32(K.pack_frames(_dev(want, cuda), d_desc, len(descs), len(blocks), got_wire, poly, total)).tolist()
    out = got_wire.cpu().numpy()
    assert np.array_equal(out[:len(wire)], wire) and (out[len(wire):] == GUARD).all(), (blens, chunk)
    assert crc4 == want_crc
    msgs, used = W.decode_stream(out[:len(wire)].tobytes())
    assert used == len(wire) and np.array_equal(np.frombuffer(b"".join(m.data for m in msgs), dtype=np.uint8), want)
    return K.u32(crc).tolist(), crc4


def _phase_segs(lens):
    """K3 segments (src_off, dst_off, len): 32 of them, every source phase twice, with source-to-destination shifts 0..15 and
    destination phases 0, 2, .., 14, 3, 7, 11, 15 -> (segs, source length, destination length)"""
    segs, pos = [], 16
    for i in range(32):
        sp = i % 16
        shift = (3 * sp) % 16 if i < 16 else (5 * sp + 1) % 16
        pos += (sp - shift - pos) % 16  # the destination phase: sp - shift
        n = lens[i % len(lens)]
        segs.append((sp + 16 * (i % 3), pos, n))
        pos += n + 1
    return segs, 32 + 15 + max(lens), pos


def _check_pages(cuda, segs, src_len, dst_len, seed):
    torch, K = _torch(), _K()
    src = _rand(src_len, seed)
    want = np.full(dst_len + SLACK, GUARD, dtype=np.uint8)
    for so, do, n in segs:
        want[do:do + n] = src[so:so + n]
    dst = _guarded(dst_len + SLACK).to(cuda)
    K.gather_pages(_dev(src, cuda), K.segs_to_device(segs, cuda), len(segs), sum(s[2] for s in segs), dst)
    got = dst.cpu().numpy()
    assert np.array_equal(got, want), [(so, do, n) for so, do, n in segs if not np.array_equal(got[do:do + n], want[do:do + n])][:4]
    return got


def _strided_case(U):
    """(src_off, dst_off, len, rows, src_pitch, dst_pitch): rows of about 2^s bytes at other pitches and phases, an empty descriptor in
    between; 3 + 4 rows, so trains of 3 rows split the second descriptor"""
    a = (5, 3, U + 3, 3, U + 37, U + 21)
    b = (0, 0, 0, 2, 8, 8)
    c_src, c_dst = 5 + 3 * (U + 37) + 11, 3 + 3 * (U + 21) + 6
    c = (c_src, c_dst, U - 7, 4, U + 1, U + 9)
    return [a, b, c], c_src + 4 * (U + 1), c_dst + 4 * (U + 9)


def _check_strided(cuda, segs, src_len, dst_len, seed):
    torch, K = _torch(), _K()
    src = _rand(src_len, seed)
    want = np.full(dst_len + SLACK, GUARD, dtype=np.uint8)
    for so, do, n, rows, sp, dp in segs:
        for r in range(rows if n else 0):
            want[do + r * dp:do + r * dp + n] = src[so + r * sp:so + r * sp + n]
    dst = _guarded(dst_len + SLACK).to(cuda)
    K.gather_strided(_dev(src, cuda), K.strided_segs_to_device(segs, cuda), len(segs), sum(s[2] * s[3] for s in segs), dst)
    got = dst.cpu().numpy()
    assert np.array_equal(got, want), [s for s in segs if s[2]]
    return got


def _check_blocks(cuda, world, bs, nb, seed):
    """deinterleave_blocks from one gathered buffer (shards at an odd stride) and gather_shards_p2p from separate local shard
    allocations, into file order; the last block is short -> the file bytes both produced"""
    torch, K = _torch(), _K()
    file_len = bs * nb - min(1000, bs // 2)
    data = _rand(file_len, seed)
    per = -(-nb // world)
    stride = per * bs + 7
    gathered = np.zeros(world * stride, dtype=np.uint8)
    shards = [np.zeros(per * bs, dtype=np.uint8) for _ in range(world)]
    for b in range(nb):
        blk = data[b * bs:(b + 1) * bs]
        o = (b // world) * bs
        gathered[(b % world) * stride + o:(b % world) * stride + o + len(blk)] = blk
        shards[b % world][o:o + len(blk)] = blk
    out = []
    dst = _guarded(file_len + SLACK).to(cuda)
    K.deinterleave_blocks(_dev(gathered, cuda), stride, world, bs, nb, file_len, dst)
    out.append(dst.cpu().numpy())
    d_shards = [_dev(s, cuda) for s in shards]
    dst = _guarded(file_len + SLACK).to(cuda)
    K.gather_shards_p2p([s.data_ptr() for s in d_shards], bs, nb, file_len, dst)
    out.append(dst.cpu().numpy())
    for got, what in zip(out, ("deinterleave", "p2p")):
        assert np.array_equal(got[:file_len], data), (what, world, bs, nb)
        assert (got[file_len:] == GUARD).all(), (what, world, bs, nb)
    return out


# ---- every launcher at every forced segment size


@pytest.mark.parametrize("poly", [0, 1])
@_seg_param()
def test_k1_crc_of_pieces_around_the_segment_size(cuda, seg, poly):
    U = 1 << seg
    _check_k1(cuda, [0, 1, 15, 16, U - 16, U - 1, U, U + 1, U + 16, 3 * U + 17], poly, 10 * seg + poly)


@_seg_param()
def test_k2_k4_frames_around_the_segment_size(cuda, seg):
    """blocks of k * 2^s +- a few bytes; frames of 2^s + 40 and of 3/4 * 2^s + 8 payload bytes, so frame edges fall inside segments
    and the 22-byte prefixes rotate the payloads' source phase"""
    U = 1 << seg
    blens = [U - 3, 2 * U + 5, 3 * U + 1, 7]
    _check_frames(cuda, blens, U + 40, 1, 20 * seg)
    _check_frames(cuda, blens, 3 * U // 4 + 8, 0, 20 * seg + 10)


@_seg_param()
def test_k3_gather_pages_every_source_phase(cuda, seg):
    U = 1 << seg
    segs, src_len, dst_len = _phase_segs([U + 17, U - 1, 9, U // 2 + 3, 2 * U + 1, U])
    _check_pages(cuda, segs, src_len, dst_len, 30 * seg)


@pytest.mark.parametrize("train", [0, 3], ids=["train_default", "train_3_rows"])
@_seg_param()
def test_gather_strided_rows_of_a_segment(cuda, seg, train, tune):
    tune(6, train)
    segs, src_len, dst_len = _strided_case(1 << seg)
    _check_strided(cuda, segs, src_len, dst_len, 40 * seg + train)


@_seg_param()
def test_deinterleave_and_p2p_gather_blocks_of_a_segment(cuda, seg):
    U = 1 << seg
    for world, bs, nb in ((2, U + 40, 4), (3, U - 24, 5)):
        _check_blocks(cuda, world, bs, nb, 50 * seg + world)


# ---- the same mixed input at every setting: byte-identical outputs and CRCs (cvk_tune's promise)

MIXED = {
    "k1": lambda cuda: _check_k1(cuda, [0, 1, 17, 4096, 4111, 65536 + 3, 200001, 524288 - 5, 1048576 + 9], 1, 7),
    "k2_k4": lambda cuda: _check_frames(cuda, [300001, 65536, 1, 524288 + 17], 100000 + 6, 1, 8),
    "gather_pages": lambda cuda: _check_pages(cuda, *_phase_segs([70001, 5, 4096, 262144 + 3, 33]), 9),
    "gather_strided": lambda cuda: _check_strided(cuda, *_strided_case(150000), 10),
    "deinterleave_p2p": lambda cuda: _check_blocks(cuda, 3, 200000 + 24, 5, 11),
}


def _same(a, b):
    if isinstance(a, np.ndarray):
        return a.tobytes() == b.tobytes()
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b


@pytest.mark.parametrize("launcher", list(MIXED))
def test_every_segment_size_gives_identical_results(cuda, tune, launcher):
    tune(5, 0)
    first = None
    for s in SHIFTS:
        tune(4, s)
        got = MIXED[launcher](cuda)
        if first is None:
            first = got
        assert _same(got, first), (launcher, s)


# ---- K1 at the segment sizes the input size chooses, with total_bytes an upper bound


def _sm_count(cuda):
    if MOCK:  # the shim's device reports CV_SIMT_EMU_SMS multiprocessors, 132 by default
        return int(os.environ.get("CV_SIMT_EMU_SMS", "132"))
    return _torch().cuda.get_device_properties(cuda).multi_processor_count


def _pick_seg_shift(total_bytes, sm_count):
    """kernels.cu's pick_seg_shift without the cvk_tune override"""
    target = total_bytes // (sm_count * 32 * 16 + 1)
    s = 14 if total_bytes >= 4 << 20 else 12
    while s < 20 and (1 << s) < target:
        s += 1
    return s


# (expected s, block size, number of blocks, bound): the bound 2^s * (32 * 16 * SMs + 1) makes the per-warp target exactly 2^s;
# None -> that bound.  The last: bench.py's K1 over its shard, 4 MiB blocks with a 16 GiB total.
DERIVED = [(14, None, 5, 8 << 20)] + [(s, None, 5, None) for s in range(15, 21)] + [(18, 4 << 20, 4, 16 << 30)]
DERIVED_IDS = ["s%d" % s for s, *_ in DERIVED[:-1]] + ["bench_4MiB_blocks_16GiB_bound_s18"]


@pytest.mark.parametrize("poly", [0, 1])
@pytest.mark.parametrize("s,bs,nb,bound", DERIVED, ids=DERIVED_IDS)
def test_k1_with_an_upper_bound_total_at_the_derived_segment_size(cuda, tune, s, bs, nb, bound, poly):
    torch, K = _torch(), _K()
    tune(4, 0)
    sms = _sm_count(cuda)
    if bound is None:
        bound = (1 << s) * (sms * 32 * 16 + 1)
    assert _pick_seg_shift(bound, sms) == s, (bound, sms)
    if bs is None:  # blocks of 2^s +- a little and several 2^s at odd offsets
        bs = 3 * (1 << s) + 5
    data = _rand(bs * nb - 12345 + 3, 60 + s + poly)
    offs = [3 + i * bs for i in range(nb)]
    lens = [min(bs, len(data) - o) for o in offs]
    assert sum(lens) <= bound
    d = _dev(data, cuda)
    dev = d.device
    offs_t = torch.tensor(offs, dtype=torch.int64, device=dev)
    lens_t = torch.tensor(lens, dtype=torch.int64, device=dev)
    out = torch.empty(nb, dtype=torch.int32, device=dev)
    K.crc_blocks_raw(d.data_ptr(), offs_t, lens_t, nb, poly, bound, out)
    got = K.u32(out).tolist()
    if bs == 4 << 20:
        assert got == clib.crc_blocks(poly, data[3:], bs).tolist()
    assert got == [clib.crc(poly, data[o:o + n]) for o, n in zip(offs, lens)]


# ---- K5 with view positions, widths and row steps past 2^32

# name -> (cols, block_rows, block_cols, view0, view_step, rows, elems).  Every segment crosses a tile edge at an element that is
# not a multiple of 8 from its start (chunks straddle it); the first two also cross a view row.  The widths are not 2^32 plus a
# small number: a scale index computed with 32-bit divisions then still lands inside the scale buffer and fails the comparison.
_C1, _C2 = (1 << 32) + (1 << 31) + 77, (1 << 32) + (1 << 31) + 1003
WIDE = {
    "view0_past_2_32": (7168, 128, 1000, (1 << 32) + 17345, 0, 1, 5000),
    "cols_past_2_32": (_C1, 1, 1 << 20, _C1 - 3003, 0, 1, 7000),
    "view0_and_cols_past_2_32": (_C2, 1, (1 << 20) + 3, _C2 + 2048 * ((1 << 20) + 3) - 3001, 0, 1, 6000),
    "view_step_past_2_32": ((1 << 31) + 5, 2, (1 << 20) - 1, 2047 * ((1 << 20) - 1) - 2500, 2 * ((1 << 31) + 5), 3, 5000),
}


def _scale_index(view0, view_step, row, elems, cols, br, bc, scols):
    """the scale each element of one segment row takes, in uint64"""
    u = np.uint64
    v = u(view0) + u(row) * u(view_step) + np.arange(elems, dtype=np.uint64)
    return (v // u(cols) // u(br)) * u(scols) + (v % u(cols)) // u(bc)


@pytest.mark.parametrize("case", list(WIDE))
def test_k5_scaled_views_past_2_32(cuda, case):
    """E4M3 and E5M2 into BF16, F16 and F32, with F32 and BF16 scales: 12 segments over the same source rows in one launch"""
    torch = _torch()
    cols, br, bc, view0, step, rows, elems = WIDE[case]
    scols = -(-cols // bc)
    idx = [_scale_index(view0, step, r, elems, cols, br, bc, scols) for r in range(rows)]
    srows = max(int(i.max()) for i in idx) // scols + 1
    rng = np.random.default_rng(list(WIDE).index(case))
    s32 = _scales(rng, srows * scols, torch.float32)
    scale_sets = {"float32": s32, "bfloat16": s32.to(torch.bfloat16)}
    d_scales = {k: v.to(cuda) for k, v in scale_sets.items()}
    pitch = elems + 9
    src = rng.integers(0, 256, size=3 + rows * pitch, dtype=np.uint8)
    segs, scales, where, at = [], [], [], 16
    for sname in F8:
        for dname in DSTS:
            for scname in scale_sets:
                sdt, ddt = getattr(torch, sname), getattr(torch, dname)
                ds = ddt.itemsize
                at += (-at) % ds + ds * (len(segs) % 5)
                dp = elems * ds + 3 * ds
                segs.append((3, at, elems, rows, pitch, dp, _code(sdt), _code(ddt)))
                scales.append((d_scales[scname].data_ptr(), _code(getattr(torch, scname)), br, bc, scols, cols, view0, step))
                where.append((at, dp, sdt, ddt, scale_sets[scname]))
                at += rows * dp + 16
    got = _scaled_on_device(cuda, np.concatenate([src, np.zeros(SLACK, dtype=np.uint8)]), segs, scales, at + SLACK)
    want = np.full(at + SLACK, GUARD, dtype=np.uint8)
    for at, dp, sdt, ddt, s in where:
        for r in range(rows):
            n = elems * ddt.itemsize
            ref = _reference(_view(src[3 + r * pitch:3 + r * pitch + elems], sdt), s, torch.from_numpy(idx[r].astype(np.int64)), ddt)
            _assert_same(_view(got[at + r * dp:at + r * dp + n], ddt), ref, (case, sdt, ddt, s.dtype, r))
            want[at + r * dp:at + r * dp + n] = got[at + r * dp:at + r * dp + n]
    assert np.array_equal(got, want), "bytes outside the destination rows were written"


def _wide_ranges():
    """(file_off, row_len, rows, file_pitch, src dtype, dst dtype, scale) as in test_zzz_readv_scaled_gpu, with scale = (dtype,
    scale_rows, scale_cols, block_rows, block_cols, cols, first_elem): a 40-row slice and a long row deep into weights of more than
    4 Gi elements, a 1-D view wider than 2^32 across a tile edge, and a plain range"""
    def rows_for(first, last_off, cols, br):
        return (first + last_off) // cols // br + 1
    c3, b3 = (1 << 32) + (1 << 31) + 1003, (1 << 20) + 3
    f1, f2, f3 = (1 << 32) + 1000, (1 << 32) + 12345, 4096 * b3 - 1000
    return [(7, 1500, 40, 3000, "float8_e4m3fn", "bfloat16", ("float32", rows_for(f1, 39 * 3000 + 1499, 3000, 128), 24, 128, 128, 3000, f1)),
            (121000, 5 * BS + 3, 1, 0, "float8_e5m2", "float32", ("bfloat16", rows_for(f2, 5 * BS + 2, 7168, 128), 56, 128, 128, 7168, f2)),
            (8 * BS + 11, 3 * BS, 1, 0, "float8_e4m3fn", "float16", ("float32", 2, -(-c3 // b3), 1, b3, c3, f3)),
            (12 * BS + 5, 2 * BS, 1, 0, "uint8", "uint8", None)]


@pytest.mark.parametrize("mode", ["files", "framed"])
def test_scaled_reads_with_view_positions_past_2_32(cuda, cluster, mode):
    torch = _torch()
    plain, _, _ = cluster
    n, ino = 24 * BS, 9990 + ["files", "framed"].index(mode)
    path = "/ls/%s" % mode
    man = plain.create_file(path, ino, n, BS, threads=2)
    want = np.frombuffer(synth.file_bytes(ino, n, BS), dtype=np.uint8)
    crcs = clib.crc_blocks(1, want, BS).astype(np.uint64)
    rng = np.random.default_rng(31)
    ranges = _wide_ranges()
    with _fs_for(cluster, mode, man, 1) as fs:
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


# (rows, cols, block_rows, block_cols): weights whose last element sits past 2^32 -- rows past 2^32 / cols elements, and cols past
# 2^32 -- with a scale grid that ends exactly at the weight's last row
GUARD_CASES = [(1 << 20, 7168, 1 << 20, 1000), (2, (1 << 32) + (1 << 31) + 5, 1, 1 << 24), (3, (1 << 32) + (1 << 31) + 9, 3, (1 << 24) + 1)]


@pytest.mark.parametrize("R,C,br,bc", GUARD_CASES, ids=["rows_2_20_cols_7168", "two_rows_cols_past_2_32", "three_rows_cols_past_2_32"])
def test_the_last_scale_of_a_wide_view_is_the_last_one_read(cuda, R, C, br, bc):
    """The weight's last elements, in partial and whole last chunks at every destination alignment: the scale walk, started from a
    view position past 2^32, reads the last scale and never the one past it (a guard page follows the scales)."""
    if not MOCK:
        pytest.skip("needs a guard page behind the scales: on the GPU a stray read would only show as a fault")
    torch = _torch()
    SR, SC = -(-R // br), -(-C // bc)
    rng = np.random.default_rng(SC)
    s = _scales(rng, SR * SC, torch.float32)
    g = _GuardedScales(s)
    try:
        last = R * C
        src = rng.integers(0, 256, size=64 + SLACK, dtype=np.uint8)
        segs, scales, where, at = [], [], [], 0
        for shift in range(8):
            for n in (1, 8 + shift, 37 + shift):
                at += (-at) % 16 + 2 * shift
                segs.append((0, at, n, 1, 0, 0, _lib.DTYPE_F8_E4M3, _lib.DTYPE_BF16))
                scales.append((g.ptr, _lib.DTYPE_F32, br, bc, SC, C, last - n, 0))
                where.append((at, n))
                at += 2 * n + 16
        got = _scaled_on_device(cuda, src, segs, scales, at + SLACK)
        for at, n in where:
            idx = _scale_index(last - n, 0, 0, n, C, br, bc, SC)
            assert int(idx[-1]) == SR * SC - 1
            _assert_same(_view(got[at:at + 2 * n], torch.bfloat16),
                         _reference(_view(src[:n], torch.float8_e4m3fn), s, torch.from_numpy(idx.astype(np.int64)), torch.bfloat16), (at, n))
    finally:
        g.close()
