"""Checkpoint loads at the size real loads run at: a safetensors checkpoint of about 0.9 GiB in 4 MiB blocks, written from HBM through
fs.create(...).write_device(...) (the K4 write path) with a 4 MiB chunk, then loaded with the benches' client configuration (16 fetch
threads, verify batches of 16, copy groups of 8, 4 MiB GPU chunks, zero-copy, arena preregistration), so the reader's 256 MiB
boundary staging runs several rounds per call.  Every tensor of every load is checked against a CPU reference: load_file() as stored,
dtype=bfloat16 / float16 against Tensor.to(), slices of ranks 0, 3 and 7 of world 8 on dim 0 and dim 1 with and without a dtype, and
FP8 weights dequantized with their block, per-row and per-tensor scales against the CPU dequant, whole and sliced.  For every call,
verify() reports no bad block, as many verified blocks as the call's ranges touch (from the header offsets) and the oracle's CRC-32C
sum over them.  One direct readv_scaled_device call puts plain, strided, cast and scaled rows at both ends of a pool of more than
4 GiB: offsets of its spans inside one range, and relative to the lowest pointer, reach past 2^32.

The arena tier runs every load; the files and framed modes run one load of each kind from the same file.  On the host-side stand-ins
(tests/simt_emu) the same checks run on a 10 MiB checkpoint in 64 KiB blocks with 48 ring slots (3 MiB of staging per round); the
pool of more than 4 GiB is host memory there, untouched but for the guarded rows."""
import json
import os
import shutil
import struct
import tempfile

import numpy as np
import pytest

from curvine_b200 import fs as F
from curvine_b200 import safetensors as ST
from oracle import clib
from test_zzz_readv_cast_gpu import GUARD, MOCK
from test_zzz_readv_scaled_gpu import _assert_same, _dequant

pytestmark = pytest.mark.gpu

BS = (64 << 10) if MOCK else (4 << 20)
PATH = "/scale/model.safetensors"
TILE = (128, 128)
WORLD, RANKS = 8, (0, 3, 7)
POOL = (4 << 30) + (64 << 20)  # one destination allocation of more than 4 GiB
# name, dtype, shape at full size, shape on the stand-ins; a 1-D norm first, so the F32 weight after it starts mid-block
SPECS = [
    ("norm.0", "float32", (4096,), (1024,)),
    ("mlp.up", "float32", (11008, 4096), (344, 1024)),
    ("embed", "bfloat16", (32003, 4096), (1003, 1024)),
    ("odd", "float16", (4096, 4099), (256, 4099)),
    ("norm.1", "bfloat16", (4099,), (1027,)),
    ("ids", "int64", (1000, 37), (100, 37)),
    ("mask", "bool", (999, 13), (99, 13)),
    ("q.weight", "float8_e4m3fn", (4100, 7000), (260, 700)),  # 128 x 128 tiles with partial edge tiles
    ("q.weight_scale_inv", "float32", (33, 55), (3, 6)),
    ("k.weight", "float8_e5m2", (3000, 5000), (300, 500)),  # per-row bfloat16 scales
    ("k.weight_scale", "bfloat16", (3000, 1), (300, 1)),
    ("o.weight", "float8_e4m3fn", (2048, 4096), (128, 256)),  # one scale for the tensor
    ("o.weight_scale", "float32", (), ()),
    ("mlp.down", "float32", (4096, 11008), (256, 1376)),
    ("lm_head", "float16", (8192, 4096), (512, 1024)),
    ("mlp.gate", "float32", (11008, 4096), (344, 1024)),  # random bits: NaNs, infinities, subnormals, rounding ties
]
SCALES = {"q.weight": "q.weight_scale_inv", "k.weight": "k.weight_scale", "o.weight": "o.weight_scale"}


def _torch():
    import torch
    return torch


def _make_tensor(torch, g, name, dt, shape):
    if dt.is_floating_point and dt.itemsize == 1:
        return torch.randint(0, 256, shape, generator=g, dtype=torch.int32).to(torch.uint8).view(dt)
    if name == "mlp.gate":
        return torch.randint(-(1 << 31), 1 << 31, shape, generator=g, dtype=torch.int64).to(torch.int32).view(torch.float32)
    if name.endswith(("_scale_inv", "_scale")):
        return (torch.rand(shape, generator=g) * 2.0 ** torch.randint(-12, 4, shape, generator=g).float()).to(dt)
    if dt.is_floating_point:
        return (torch.randn(shape, generator=g) * 300).to(dt)
    return torch.randint(0, 2 if dt == torch.bool else 1 << 40, shape, generator=g).to(dt)


class Checkpoint:
    """the tensors (CPU views into `blob`, the file's bytes), the header, and the oracle's per-block CRCs"""

    def __init__(self):
        torch = _torch()
        g = torch.Generator().manual_seed(29)
        names = {v: k for k, v in ST.dtypes().items()}
        made, header, off = [], {}, 0
        for name, dt_name, full, small in SPECS:
            dt = getattr(torch, dt_name)
            t = _make_tensor(torch, g, name, dt, small if MOCK else full)
            off += -off % dt.itemsize  # converted tensors sit at multiples of their element size
            header[name] = {"dtype": names[dt], "shape": list(t.shape), "data_offsets": [off, off + t.numel() * dt.itemsize]}
            made.append((name, t, off))
            off += t.numel() * dt.itemsize
        raw = json.dumps(header).encode()
        raw += b" " * (-(8 + len(raw)) % 8)
        self.start = 8 + len(raw)
        self.blob = np.zeros(self.start + off, dtype=np.uint8)
        self.blob[:self.start] = np.frombuffer(struct.pack("<Q", len(raw)) + raw, dtype=np.uint8)
        self.tensors = {}
        for name, t, o in made:
            n = t.numel() * t.dtype.itemsize
            self.blob[self.start + o:self.start + o + n] = t.reshape(-1).view(torch.uint8).numpy()
            self.tensors[name] = torch.from_numpy(self.blob[self.start + o:self.start + o + n]).view(t.dtype).reshape(t.shape)
        del made
        self.n = self.blob.size
        self.nb = -(-self.n // BS)
        _, self.entries = ST.parse_header(lambda o, k: self.blob[o:o + k].tobytes(), self.n)
        self.crc32 = clib.crc_blocks(0, self.blob, BS)
        self.crc32c = clib.crc_blocks(1, self.blob, BS).astype(np.uint64)

    def touched(self, ranges):
        """bool per block: touched by a row of one of `ranges` (file_off, row_len, rows, file_pitch)"""
        mark = np.zeros(self.nb + 1, dtype=np.int64)
        for off, L, R, P in ranges:
            if L and R:
                s = off + np.arange(R, dtype=np.int64) * P
                np.add.at(mark, s // BS, 1)
                np.add.at(mark, (s + L - 1) // BS + 1, -1)
        return np.cumsum(mark)[:self.nb] > 0


def _conf(mode, d):
    if MOCK:  # 48 ring slots of 64 KiB blocks: 3 MiB of staging per round
        b200 = 'fetch_threads = 2\nverify_batch = 8\ncopy_group = 8\ngpu_chunk_size = "64KB"\nzero_copy = true\n'
    else:  # the benches' configuration: 176 ring slots, so a round stages 256 MiB
        b200 = 'fetch_threads = 16\nverify_batch = 16\ncopy_group = 8\ngpu_chunk_size = "4MB"\nzero_copy = true\n'
    if mode == "arena":
        b200 += 'register_threads = 16\narena_register_slice = "%s"\narena_preregister = ["%s/arena"]\n' % ("4MB" if MOCK else "256MB", d)
    return F.client_conf(short_circuit=mode != "framed", b200=b200)


@pytest.fixture(scope="module")
def written(cuda):
    """the checkpoint, written from HBM into a plain worker and into a mem-arena worker"""
    torch = _torch()
    ck = Checkpoint()
    d = tempfile.mkdtemp(prefix="cvsc", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    seg = (8 << 20) if MOCK else (256 << 20)
    plain = F.MiniWorker(["[MEM]" + d + "/mem"])
    arena = F.MiniWorker(["[MEM:%d]%s/arena" % ((ck.n + BS + seg - 1) // seg * seg + seg, d)],
                         extra_worker='mem_arena = true\narena_segment = "%d"\narena_reuse_delay = "0ms"\n' % seg)
    try:
        hbm = torch.from_numpy(ck.blob).to(cuda)
        mans = {}
        with F.CurvineFileSystem(F.client_conf(short_circuit=False)) as wfs:
            for key, w in (("plain", plain), ("arena", arena)):
                wr = wfs.create(PATH, 7700 + len(mans), BS, w.port, chunk_size=BS)
                wr.write_device(hbm.data_ptr(), ck.n, torch.cuda.current_stream().cuda_stream)
                mans[key] = wr.complete()
        del hbm
        for man in mans.values():  # the manifest's block CRCs, computed on the GPU while writing, equal the oracle's over the file bytes
            blocks = [line.split() for line in man.splitlines() if line.startswith("block ")]
            assert [int(b[2]) for b in blocks] == [min(BS, ck.n - i * BS) for i in range(ck.nb)]
            assert [int(b[4], 16) for b in blocks] == [int(x) for x in ck.crc32]
            assert [int(b[5], 16) for b in blocks] == [int(x) for x in ck.crc32c]
        yield ck, mans, d
    finally:
        plain.stop()
        arena.stop()
        shutil.rmtree(d, ignore_errors=True)


@pytest.fixture(scope="module", params=["arena", "files", "framed"])
def mode_fs(request, written):
    ck, mans, d = written
    mode = request.param
    with F.CurvineFileSystem(_conf(mode, d)) as fs:
        fs.load_namespace(mans["arena" if mode == "arena" else "plain"])
        if mode == "arena":
            fs.preregister()
            fs.wait_registered()
        yield mode, fs, ck


@pytest.fixture
def verified(monkeypatch):
    """every verify() result of the loads: load_file calls verify() itself"""
    calls = []
    orig = F.Reader.verify

    def spy(self):
        out = orig(self)
        calls.append(out)
        return out
    monkeypatch.setattr(F.Reader, "verify", spy)
    return calls


def _floats(torch):
    return (torch.float32, torch.float16, torch.bfloat16)


def _expect(ck, name, dtype, scales, sl):
    torch = _torch()
    t = ck.tensors[name]
    if scales and name in scales:
        w = _dequant(t, ck.tensors[scales[name]], TILE, dtype)
    elif dtype is not None and t.dtype in _floats(torch):
        w = t.to(dtype)
    else:
        w = t
    if sl and name in sl:
        dim, a, b = sl[name]
        w = w.narrow(dim, a, b - a)
    return w.contiguous()


def _same(got, want, what):
    torch = _torch()
    assert got.dtype == want.dtype and tuple(got.shape) == tuple(want.shape), (what, got.dtype, tuple(got.shape), want.dtype, tuple(want.shape))
    w = want.reshape(-1).to(got.device)
    if want.dtype in _floats(torch):
        _assert_same(got.reshape(-1), w, what)
    else:
        assert torch.equal(got.reshape(-1).view(torch.uint8), w.view(torch.uint8)), what


def _load(fs, ck, verified, cuda, names, **kw):
    """load_file(**kw), every tensor against its CPU reference, and the call's verify() against the blocks its ranges touch"""
    torch = _torch()
    dev = "cpu" if MOCK else cuda
    verified.clear()
    got = ST.load_file(fs, PATH, device=dev, names=names, **kw)
    torch.cuda.synchronize()
    assert len(verified) == 1
    plan = ST.plan_ranges(ck.start, ck.entries, names, kw.get("slices"), kw.get("dtype"), kw.get("scales"), kw.get("scale_block"))
    blocks = [ck.touched([r[:4] for *_, r in plan if r is not None])]
    if kw.get("scales"):  # the first call reads every scale a selected weight uses, whole and as stored
        used = dict.fromkeys(r[7][0] for *_, r in plan if r is not None and r[7] is not None)
        blocks.append(ck.touched([(ck.start + ck.entries[s][2], ck.entries[s][3] - ck.entries[s][2], 1, 0) for s in used]))
    s, bad, ver = verified[0]
    assert bad == 0 and ver == sum(int(b.sum()) for b in blocks), (ver, [int(b.sum()) for b in blocks], kw)
    assert s == sum(int(ck.crc32c[b].sum()) for b in blocks), kw
    assert list(got) == list(names)
    for name in names:
        _same(got[name], _expect(ck, name, kw.get("dtype"), kw.get("scales"), kw.get("slices")), (name, kw))
        del got[name]
    return plan


def _rank_slices(ck, dim, rank):
    return {name: (dim, rank * t.shape[dim] // WORLD, (rank + 1) * t.shape[dim] // WORLD) for name, t in ck.tensors.items() if t.dim() == 2}


def _not_fp8(ck):
    return [n for n, t in ck.tensors.items() if t.dtype.itemsize != 1 or not t.dtype.is_floating_point]


def test_the_cast_load_runs_several_staging_rounds(cuda, mode_fs):
    """the file's converting tensors need more than two rounds of the reader's staging (at most 64 blocks of 4 MiB)"""
    mode, fs, ck = mode_fs
    torch = _torch()
    plan = ST.plan_ranges(ck.start, ck.entries, _not_fp8(ck), dtype=torch.bfloat16)
    with fs.open(PATH) as r:
        spans, _, _ = r.readv_cast_plan([x[:4] + (0,) + x[4:] for *_, x in plan if x is not None])
    staged = {sp[0] for sp in spans if not sp[5]}
    per_round = min(48 if MOCK else 176, (256 << 20) // BS)
    assert len(staged) > 2 * per_round, (len(staged), per_round)


@pytest.mark.parametrize("dtype", [None, "bfloat16", "float16"])
def test_whole_loads(cuda, mode_fs, verified, dtype):
    mode, fs, ck = mode_fs
    torch = _torch()
    if mode != "arena" and dtype != "bfloat16":
        pytest.skip("the files and framed modes run one load of each kind")
    dt = getattr(torch, dtype) if dtype else None
    _load(fs, ck, verified, cuda, list(ck.tensors) if dt is None else _not_fp8(ck), dtype=dt)


@pytest.mark.parametrize("dtype", [None, "bfloat16"])
@pytest.mark.parametrize("dim", [0, 1])
def test_tensor_parallel_slices(cuda, mode_fs, verified, dim, dtype):
    mode, fs, ck = mode_fs
    torch = _torch()
    if mode != "arena" and (dim, dtype) != (1, "bfloat16"):
        pytest.skip("the files and framed modes run one load of each kind")
    dt = getattr(torch, dtype) if dtype else None
    for rank in RANKS if mode == "arena" else (3,):
        names = list(ck.tensors) if dt is None else _not_fp8(ck)
        sl = {k: v for k, v in _rank_slices(ck, dim, rank).items() if k in names}
        _load(fs, ck, verified, cuda, names, slices=sl, dtype=dt)


@pytest.mark.parametrize("sliced", [False, True])
def test_fp8_dequantized_loads(cuda, mode_fs, verified, sliced):
    mode, fs, ck = mode_fs
    torch = _torch()
    if mode != "arena" and sliced:
        pytest.skip("the files and framed modes run one load of each kind")
    for dim, rank in [(d, r) for d in (0, 1) for r in RANKS] if sliced else [(None, None)]:
        sl = _rank_slices(ck, dim, rank) if sliced else None
        _load(fs, ck, verified, cuda, list(ck.tensors), slices=sl, dtype=torch.bfloat16, scales=SCALES, scale_block=TILE)


def test_destinations_more_than_4_gib_apart(cuda, written):
    """one readv_scaled_device call into one pool of POOL bytes: a plain range of whole blocks at its start, and a strided plain, a
    cast and a scaled range whose row 0 lies near the pool's start and row 1 near its end (dst_pitch > 4 GiB, row 1 in another block)"""
    torch = _torch()
    ck, mans, d = written
    e = ck.entries
    q0, C, R = ck.start + e["q.weight"][2], ck.tensors["q.weight"].shape[1], ck.tensors["q.weight"].shape[0]
    step = -(-BS // C) + 1  # weight rows between the range's two rows: they lie in different blocks
    r0 = R // 3
    up0 = ck.start + e["mlp.up"][2]
    mib = 1 << 20
    # (file_off, row_len, rows, file_pitch, dst offset in the pool, dst_pitch, src dtype, dst dtype, scale)
    ranges = [((ck.nb - 3) * BS, 2 * BS, 1, 0, 0, 0, "uint8", "uint8", None),  # two whole blocks of mlp.gate: direct
              (ck.start + e["embed"][2] + 777, 3000, 2, 2 * BS + 100, 16 * mib + 5, POOL - 32 * mib, "uint8", "uint8", None),
              (up0 + 4 * 1001, BS + 1236, 2, 3 * BS + 8, 32 * mib + 2, POOL - 64 * mib, "float32", "bfloat16", None),
              (q0 + r0 * C, 2 * C, 2, step * C, 48 * mib, POOL - 96 * mib, "float8_e4m3fn", "bfloat16", "q")]
    s_q = ck.tensors["q.weight_scale_inv"]
    d_s = s_q.to(cuda)
    pool = torch.empty(POOL, dtype=torch.uint8, device=cuda)
    rows = []  # (pool offset, bytes, expected bytes or (expected tensor))
    for off, L, nr, P, at, dp, sn, dn, sc in ranges:
        sdt, ddt = getattr(torch, sn), getattr(torch, dn)
        for k in range(nr):
            src = torch.from_numpy(ck.blob[off + k * P:off + k * P + L])
            if sc:
                v = r0 * C + k * step * C + torch.arange(L)
                idx = (v // C // TILE[0]) * s_q.shape[1] + (v % C) // TILE[1]
                want = (src.view(sdt).float() * s_q.reshape(-1)[idx]).to(ddt)
            else:
                want = src.view(sdt).to(ddt)
            rows.append((at + k * dp, want))
            n = want.numel() * ddt.itemsize
            pool[at + k * dp - (64 if at + k * dp else 0):at + k * dp + n + 64].fill_(GUARD)  # guard bytes around the rows only
    call = [(off, L, nr, P, pool.data_ptr() + at, dp, getattr(torch, sn), getattr(torch, dn),
             (d_s.data_ptr(), torch.float32, s_q.shape[0], s_q.shape[1], TILE[0], TILE[1], C, r0 * C) if sc else None)
            for off, L, nr, P, at, dp, sn, dn, sc in ranges]
    with F.CurvineFileSystem(_conf("arena", d)) as fs:
        fs.load_namespace(mans["arena"])
        r = fs.open(PATH)
        got = r.readv_scaled_device(call, torch.cuda.current_stream().cuda_stream)
        s, bad, ver = r.verify()
        torch.cuda.synchronize()
        r.complete()
    assert got == sum(w.numel() * w.dtype.itemsize for _, w in rows)
    top = max(at + w.numel() * w.dtype.itemsize for at, w in rows)
    print("largest destination offset from the pool's start: %d bytes (2^32 + %d)" % (top, top - (1 << 32)))
    assert top > (1 << 32) + (16 << 20)
    for at, want in rows:
        n = want.numel() * want.dtype.itemsize
        row = pool[at:at + n]
        if want.dtype == torch.uint8:
            assert torch.equal(row, want.to(cuda)), at
        else:
            _assert_same(row.view(want.dtype), want.to(cuda), at)
        if at:
            assert bool((pool[at - 64:at] == GUARD).all()), at
        assert bool((pool[at + n:at + n + 64] == GUARD).all()), at
    touched = ck.touched([x[:4] for x in ranges])
    assert bad == 0 and ver == int(touched.sum()) and s == int(ck.crc32c[touched].sum())
