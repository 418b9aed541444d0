"""Checkpoints the official safetensors writer produced, loaded on the GPU and checked against a plain numpy reference.

The files are those of tests/golden/safetensors_official.json (FP8 weights with F32 / F16 / BF16 scales per tensor, per row and in
block grids of (128, 128), (1, 16), (3, 7) and (64, 48); float tensors salted with cast edges; integer, bool, empty and 0-d tensors
between them; F8_E8M0, F4 and C64 tensors), rebuilt byte for byte and written through fs.create(...).write() at block sizes of 12292
and 65540 bytes (multiples of 4 but of neither 16 nor 4096, so block edges fall inside rows, scale tiles and K5's 8-element chunks)
and 32768 bytes.  Every load runs in the files, framed and arena modes with copy groups of 1 and 4: whole loads, name subsets (a
scale tensor without its weight among them), dtype None / float32 / float16 / bfloat16, and the slices of every rank of worlds 2, 3
and 8 on dims 0, 1 and -1, composed with scales= / scale_block=.

The reference knows nothing of torch's conversions: FP8 bytes decode through 256-entry float64 tables built from the format
definitions, scales and float tensors decode by bit view, the exact float64 product rounds once to float32 (numpy) and then to float16
(numpy) or bfloat16 (integer round-to-nearest-even on the float32 bits).  A NaN only has to stay a NaN.  Every load's verify() must
report no bad block, as many verified blocks as the selected bytes (and, for the scales' own read, the scale tensors) touch, and the
oracle's CRC-32C sum over them.  On the host-side stand-ins (tests/simt_emu) one block size and every third load run."""
import json
import os
import shutil
import struct
import tempfile

import numpy as np
import pytest

from curvine_b200 import fs as F
from curvine_b200 import safetensors as ST
from oracle import clib, layout
from test_safetensors_format import CKS, RECORD, official_file
from test_zzz_readv_cast_gpu import MOCK, _fs_for

pytestmark = pytest.mark.gpu

BLOCKS = [12292] if MOCK else [12292, 65540, 32768]
FLOATS = ("float32", "float16", "bfloat16")


def _torch():
    import torch
    return torch


# ---- the reference

def _fp8_table(fmt):
    """float64 value of each of the 256 bytes of F8_E4M3 (E4M3FN: bias 7, no infinities, S.1111.111 is NaN) or F8_E5M2 (bias 15,
    IEEE-like: exponent 31 is infinity or NaN)"""
    b = np.arange(256)
    sign = np.where(b >> 7, -1.0, 1.0)
    if fmt == "F8_E4M3":
        e, m, bias, mb = (b >> 3) & 15, b & 7, 7, 3
    else:
        e, m, bias, mb = (b >> 2) & 31, b & 3, 15, 2
    frac = m / float(1 << mb)
    v = sign * np.where(e == 0, frac * 2.0 ** (1 - bias), (1 + frac) * 2.0 ** (e - bias))
    if fmt == "F8_E4M3":
        v[(e == 15) & (m == 7)] = np.nan
    else:
        v[(e == 31) & (m == 0)] = sign[(e == 31) & (m == 0)] * np.inf
        v[(e == 31) & (m != 0)] = np.nan
    return v


TABLES = {f: _fp8_table(f) for f in ("F8_E4M3", "F8_E5M2")}
UINT = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}


def decode(raw, dt):
    """the stored bytes of a F32 / F16 / BF16 / F8_* tensor -> float64 values"""
    with np.errstate(invalid="ignore"):
        return _decode(raw, dt)


def _decode(raw, dt):
    if dt in TABLES:
        return TABLES[dt][np.frombuffer(raw, dtype=np.uint8)]
    if dt == "F32":
        return np.frombuffer(raw, dtype=np.float32).astype(np.float64)
    if dt == "F16":
        return np.frombuffer(raw, dtype=np.float16).astype(np.float64)
    return (np.frombuffer(raw, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def round_to(x, target):
    """float64 values -> (bits of `target`, NaN mask): one rounding to float32, then one to the result dtype"""
    with np.errstate(over="ignore", invalid="ignore"):
        f32 = x.astype(np.float32)
        if target == "float32":
            bits = f32.view(np.uint32)
        elif target == "float16":
            bits = f32.astype(np.float16).view(np.uint16)
        else:
            u = f32.view(np.uint32).astype(np.uint64)
            bits = (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) & 0xFFFF).astype(np.uint16)
    return bits, np.isnan(x)


def _scale_index(shape, sshape, block):
    """per element of a weight of `shape`, the flat index of its scale in a scale tensor of `sshape`"""
    n = int(np.prod(shape, dtype=np.int64))
    cols = shape[-1] if shape else 1
    v = np.arange(n, dtype=np.int64)
    r, c = v // max(cols, 1), v % max(cols, 1)
    if int(np.prod(sshape, dtype=np.int64)) == 1:
        return np.zeros(n, dtype=np.int64)
    if tuple(sshape) == (shape[0], 1):
        return r
    return (r // block[0]) * sshape[1] + c // block[1]


# what the reference needs of each dtype the checkpoints load: bytes per element and the torch dtype of the result as stored
ITEMSIZE = {"F8_E4M3": 1, "F8_E5M2": 1, "F8_E8M0": 1, "F32": 4, "F16": 2, "BF16": 2, "I64": 8, "I32": 4, "U16": 2, "U8": 1, "BOOL": 1,
            "C64": 8}
TORCH_NAME = {"F8_E4M3": "float8_e4m3fn", "F8_E5M2": "float8_e5m2", "F8_E8M0": "float8_e8m0fnu", "F32": "float32", "F16": "float16",
              "BF16": "bfloat16", "I64": "int64", "I32": "int32", "U16": "uint16", "U8": "uint8", "BOOL": "bool", "C64": "complex64"}


class Reference:
    """expected results of one official checkpoint, tensor by tensor, as (bits array of the result's shape, NaN mask or None).  Offsets,
    shapes and dtypes come from the recorded header JSON, not from the parser under test."""

    def __init__(self, ck):
        self.ck, self.blob = ck, official_file(ck)
        (n,) = struct.unpack("<Q", self.blob[:8])
        self.start = 8 + n
        self.hdr = {name: (e["dtype"], tuple(e["shape"]), e["data_offsets"][0], e["data_offsets"][1])
                    for name, e in json.loads(self.blob[8:self.start]).items() if name != "__metadata__"}
        spec = RECORD[ck]["spec"]
        self.scales, self.block = spec["scales"], tuple(spec["scale_block"])
        self.loadable = [name for name, (dt, *_) in self.hdr.items() if dt in ITEMSIZE]
        self._memo = {}

    def torch_dtype(self, name):
        return getattr(_torch(), TORCH_NAME[self.hdr[name][0]])

    def raw(self, name):
        _, _, b, e = self.hdr[name]
        return self.blob[self.start + b:self.start + e]

    def full(self, name, dtype, scaled):
        key = (name, dtype, scaled)
        if key not in self._memo:
            dt, shape, _, _ = self.hdr[name]
            if scaled:
                s = self.scales[name]
                with np.errstate(invalid="ignore"):  # infinity times zero: NaN
                    x = decode(self.raw(name), dt) * decode(self.raw(s), self.hdr[s][0])[_scale_index(shape, self.hdr[s][1], self.block)]
                bits, nan = round_to(x, dtype)
            elif dtype is not None and dt in ("F32", "F16", "BF16"):
                bits, nan = round_to(decode(self.raw(name), dt), dtype)
            else:  # as stored: the bytes
                bits, nan = np.frombuffer(self.raw(name), dtype=UINT[ITEMSIZE[dt]]), None
            self._memo[key] = (bits.reshape(shape), None if nan is None else nan.reshape(shape))
        return self._memo[key]

    def expect(self, name, dtype, scales, slices):
        bits, nan = self.full(name, dtype, bool(scales) and name in scales)
        if slices and name in slices:
            d, a, z = slices[name]
            bits = np.take(bits, np.arange(a, z), axis=d)
            nan = None if nan is None else np.take(nan, np.arange(a, z), axis=d)
        return bits, nan

    def touched(self, bs, names, slices, scales):
        """(blocks the load's ranges touch, blocks the scales' own read touches), from the data offsets, the slices and the scales"""
        main, sc = set(), set()
        for name in names:
            dt, shape, b, _ = self.hdr[name]
            size = ITEMSIZE[dt]
            grid = np.arange(int(np.prod(shape, dtype=np.int64)), dtype=np.int64).reshape(shape)
            if slices and name in slices:
                d, a, z = slices[name]
                grid = np.take(grid, np.arange(a, z), axis=d)
            if grid.size == 0:
                continue
            off = self.start + b + grid.ravel() * size
            main.update(np.unique(np.concatenate([off, off + size - 1]) // bs).tolist())
            if scales and name in scales:
                _, _, sb, se = self.hdr[scales[name]]
                sc.update(range((self.start + sb) // bs, (self.start + se - 1) // bs + 1))
        return sorted(main), sorted(sc)


_REFS = {}


def _ref(ck):
    if ck not in _REFS:
        _REFS[ck] = Reference(ck)
    return _REFS[ck]


def test_the_reference_equals_torch_on_the_cpu_for_every_fp8_byte():
    """every FP8 byte times a sample of scales of each scale dtype into every result dtype, and every F16 / BF16 pattern and a float32
    sample into the other float dtypes: the numpy reference and torch's CPU conversions agree, so a disagreement on the GPU says
    which side is wrong"""
    torch = _torch()
    rng = np.random.default_rng(4)
    raw = np.arange(256, dtype=np.uint8)
    f32 = np.concatenate([np.ldexp(rng.uniform(0.5, 1, 200), rng.integers(-30, 30, 200)), [0.0, -0.0, 1.0, 2.0 ** -24, 65504.0, -3e38]])
    sdt = {"F32": torch.float32, "F16": torch.float16, "BF16": torch.bfloat16}
    for fmt, tdt in (("F8_E4M3", torch.float8_e4m3fn), ("F8_E5M2", torch.float8_e5m2)):
        x = torch.from_numpy(raw.copy()).view(tdt)
        for sname, st in sdt.items():
            s = torch.from_numpy(f32).to(st)
            s_raw = s.view({4: torch.int32, 2: torch.int16}[st.itemsize]).numpy().tobytes()
            for target in FLOATS:
                tt = getattr(torch, target)
                want = (x.float()[:, None] * s.float()[None, :]).to(tt)
                with np.errstate(invalid="ignore"):
                    bits, nan = round_to(decode(raw.tobytes(), fmt)[:, None] * decode(s_raw, sname)[None, :], target)
                _check(want, bits, nan, (fmt, sname, target))
    for src in FLOATS:
        st = getattr(torch, src)
        if st.itemsize == 2:
            pat = np.arange(1 << 16, dtype=np.uint16)
        else:
            pat = np.concatenate([rng.integers(0, 1 << 32, 1 << 16, dtype=np.uint64).astype(np.uint32),
                                  np.array([0x3F808000, 0x3F818000, 0x477FF000, 0x387FF000, 0x33000000, 0x7F7FFFFF, 0x7F800001], np.uint32)])
        t = torch.from_numpy(pat.view({2: np.int16, 4: np.int32}[st.itemsize]).copy()).view(st)
        for target in FLOATS:
            bits, nan = round_to(decode(pat.tobytes(), {"float32": "F32", "float16": "F16", "bfloat16": "BF16"}[src]), target)
            _check(t.to(getattr(torch, target)), bits, nan, (src, target))


def _bits_of(t):
    torch = _torch()
    t = t.detach().cpu().contiguous()
    ints = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}
    return t.view(ints[t.dtype.itemsize]).numpy().view(UINT[t.dtype.itemsize]).reshape(tuple(t.shape))


def _check(got, bits, nan, what):
    """got (a tensor) == the reference bit for bit; where the reference is NaN, got only has to be NaN"""
    torch = _torch()
    g = _bits_of(got)
    assert g.shape == bits.shape, (what, g.shape, bits.shape)
    if nan is None:
        assert np.array_equal(g, bits), what
        return
    bad = (g != bits) & ~nan
    assert not bad.any(), (what, int(bad.sum()), g[bad][:8], bits[bad][:8])
    if nan.any():
        gf = got.detach().cpu().reshape(tuple(g.shape)).float().numpy()
        assert np.isnan(gf[nan]).all(), what


# ---- the loads

# (dtype, scales=) of the sliced loads, in turn: as stored, each cast, and each dequantization
SLICED_KINDS = [(None, False)] + [(t, False) for t in FLOATS] + [(t, True) for t in FLOATS]


def _loads(ref):
    """the deterministic load cases of one checkpoint: kwargs of load_file"""
    torch = _torch()
    rng = np.random.default_rng(sum(map(ord, ref.ck)))
    dt_of = {n: ref.hdr[n][0] for n in ref.loadable}
    plain = [n for n in ref.loadable if dt_of[n] not in ("F8_E4M3", "F8_E5M2", "F8_E8M0")]
    scaled = [n for n in ref.loadable if dt_of[n] != "F8_E8M0"]
    out = [dict(names=ref.loadable)]
    for target in FLOATS:
        dt = getattr(torch, target)
        out.append(dict(names=plain, dtype=dt))
        out.append(dict(names=scaled, dtype=dt, scales=ref.scales, scale_block=ref.block))
    lone = sorted(ref.scales.values())[0]  # a scale tensor without its weight, as stored and converted
    others = [n for n in plain if n != lone]
    sub = sorted(rng.choice(others, size=min(4, len(others)), replace=False).tolist())
    out.append(dict(names=[lone] + sub + [n for n in ref.loadable if n not in plain][:2]))
    out.append(dict(names=[lone] + sub, dtype=torch.bfloat16))
    w = sorted(ref.scales)[0]
    out.append(dict(names=[w, lone] + sub, dtype=torch.float16, scales={w: ref.scales[w]}, scale_block=ref.block))
    k = 0
    for world in (2, 3, 8):
        for dim in (0, 1, -1):
            for rank in range(world):
                target, with_scales = SLICED_KINDS[k % len(SLICED_KINDS)]
                k += 1
                names = ref.loadable if target is None else scaled if with_scales else plain
                sl = {}
                for n in names:
                    shape = ref.hdr[n][1]
                    if -len(shape) <= dim < len(shape):
                        size = shape[dim]
                        sl[n] = (dim, rank * size // world, (rank + 1) * size // world)
                kw = dict(names=names, slices=sl)
                if target is not None:
                    kw["dtype"] = getattr(torch, target)
                if with_scales:
                    kw.update(scales=ref.scales, scale_block=ref.block)
                out.append(kw)
    return out[::3] if MOCK else out  # a stride prime to the 7 kinds the sliced loads cycle through


@pytest.fixture(scope="module")
def written(cuda):
    """every official checkpoint at every block size, written through fs.create(...).write() into a plain and a mem-arena worker"""
    d = tempfile.mkdtemp(prefix="cvoi", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    plain = F.MiniWorker(["[MEM]" + d + "/mem"])
    arena = F.MiniWorker(["[MEM:64MB]" + d + "/arena"], extra_worker='mem_arena = true\narena_segment = "8MB"\n')
    try:
        mans = {"plain": [], "arena": []}
        crcs = {}
        with F.CurvineFileSystem(F.client_conf(short_circuit=False)) as wfs:
            for i, bs in enumerate(BLOCKS):
                for j, ck in enumerate(CKS):
                    blob = official_file(ck)
                    crcs[(ck, bs)] = clib.crc_blocks(1, np.frombuffer(blob, dtype=np.uint8), bs).astype(np.uint64)
                    for key, w in (("plain", plain), ("arena", arena)):
                        wr = wfs.create("/oi/%d/%s" % (bs, ck), 8400 + 10 * i + j, bs, w.port, chunk_size=8192)
                        wr.write(blob)
                        mans[key].append(wr.complete())
        yield (plain, arena, d), {k: "".join(v) for k, v in mans.items()}, crcs
    finally:
        plain.stop()
        arena.stop()
        shutil.rmtree(d, ignore_errors=True)


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


def _run_load(fs, path, ref, bs, crcs, verified, kw, dev):
    torch = _torch()
    verified.clear()
    got = ST.load_file(fs, path, device=dev, **kw)
    torch.cuda.synchronize()
    assert list(got) == list(kw["names"])
    for name in kw["names"]:
        bits, nan = ref.expect(name, _name_of(kw.get("dtype")) if kw.get("dtype") is not None else None, kw.get("scales"), kw.get("slices"))
        t = got[name]
        stored = ref.torch_dtype(name)
        want_dt = stored if kw.get("dtype") is None or (stored not in _float_dtypes() and not (kw.get("scales") and name in kw["scales"])) else kw["dtype"]
        assert t.dtype == want_dt and t.is_contiguous(), (name, t.dtype, want_dt)
        _check(t, bits, nan, (ref.ck, bs, name, kw.get("dtype"), kw.get("slices", {}).get(name), bool(kw.get("scales"))))
    main, sc = ref.touched(bs, kw["names"], kw.get("slices"), kw.get("scales"))
    assert len(verified) == 1
    s, bad, ver = verified[0]
    assert bad == 0 and ver == len(main) + len(sc), (ver, main, sc)
    assert s == int(crcs[main].sum()) + int(crcs[sc].sum())


def _float_dtypes():
    torch = _torch()
    return (torch.float32, torch.float16, torch.bfloat16)


def _name_of(dt):
    return str(dt).split(".")[-1]


@pytest.mark.parametrize("bs", BLOCKS)
@pytest.mark.parametrize("copy_group", [1, 4])
@pytest.mark.parametrize("mode", ["files", "framed", "arena"])
def test_official_checkpoints_load_as_the_numpy_reference(cuda, written, verified, mode, copy_group, bs):
    cluster, mans, crcs = written
    dev = "cpu" if MOCK else cuda
    n = 0
    with _fs_for(cluster, mode, mans["arena" if mode == "arena" else "plain"], copy_group) as fs:
        for ck in CKS:
            ref = _ref(ck)
            for kw in _loads(ref):
                _run_load(fs, "/oi/%d/%s" % (bs, ck), ref, bs, crcs[(ck, bs)], verified, kw, dev)
                n += 1
    print("%s copy_group %d block %d: %d loads" % (mode, copy_group, bs, n))


def _flip(d, worker, ino, blk, off):
    """flip one byte of block `blk` of the file of inode `ino` where the worker stores it: a block file, or an arena extent"""
    root = "%s/%s/curvine" % (d, worker)
    p = layout.block_path(root, layout.create_block_id(ino, blk))
    with open(p, "rb") as f:
        head = f.read(8)
    if head == b"CVARENA1":
        _, seg, at, _ = open(p).read().split()
        p, off = "%s/arena/seg_%04d" % (root, int(seg)), int(at) + off
    with open(p, "r+b") as f:
        f.seek(off)
        b = f.read(1)
        f.seek(off)
        f.write(bytes([b[0] ^ 0x20]))


@pytest.mark.parametrize("mode", ["files", "framed", "arena"])
def test_a_flipped_byte_fails_the_load_only_in_a_block_it_touches(cuda, written, verified, mode):
    torch = _torch()
    (plain, arena, d), _, _ = written
    dev = "cpu" if MOCK else cuda
    ck, bs, ino = "tiles_3x7", 12292, 8490 + ["files", "framed", "arena"].index(mode)
    ref = _ref(ck)
    w, wname = (arena, "arena") if mode == "arena" else (plain, "mem")
    path = "/oi/bad/%s" % mode
    with F.CurvineFileSystem(F.client_conf(short_circuit=False)) as wfs:
        wr = wfs.create(path, ino, bs, w.port, chunk_size=8192)
        wr.write(ref.blob)
        man = wr.complete()
    crcs = clib.crc_blocks(1, np.frombuffer(ref.blob, dtype=np.uint8), bs).astype(np.uint64)
    kw = dict(names=["h.bf16"], dtype=torch.float32)
    main, _ = ref.touched(bs, kw["names"], None, None)
    nb = -(-len(ref.blob) // bs)
    untouched = [b for b in range(1, nb) if b not in main]
    assert main and untouched
    _flip(d, wname, ino, untouched[-1], 100)
    with _fs_for((plain, arena, d), mode, man, 1) as fs:
        _run_load(fs, path, ref, bs, crcs, verified, kw, dev)
    at = _neighbour_byte(ref, "h.bf16", bs)
    _flip(d, wname, ino, at // bs, at % bs)
    with _fs_for((plain, arena, d), mode, man, 1) as fs:
        with pytest.raises(IOError, match="1 blocks of .* failed CRC verification"):
            ST.load_file(fs, path, device=dev, **kw)


def _neighbour_byte(ref, name, bs):
    """a file offset in a block tensor `name` touches that belongs to neither the header nor `name`: the first byte after the tensor,
    else the last one before it.  Flipping it shows that a touched block is verified whole, not only the bytes the load wants."""
    _, _, b, e = ref.hdr[name]
    b, e = ref.start + b, ref.start + e
    for at in (e, b - 1):
        if ref.start <= at < len(ref.blob) and at // bs in (b // bs, (e - 1) // bs):
            assert not b <= at < e
            return at
    raise AssertionError("%s shares no block with another tensor at block size %d" % (name, bs))
