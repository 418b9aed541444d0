"""The safetensors header parser against files the format's official writer produced, without a GPU.

The checkpoints of tests/golden/safetensors_official.json are rebuilt from their recorded headers and seeded contents, and must hash
to what safetensors.torch.save wrote.  parse_header must read every one as its header states, and as the official reader does when
the `safetensors` package is importable; it must accept every dtype name of the format and reject a shape that does not need exactly
its bytes.  Tensors of a dtype torch cannot hold (F4, F6_*) stay in the header table but cannot be loaded, and plan_ranges on these
files reads exactly the bytes a numpy restatement of each slice selects."""
import hashlib
import importlib.util
import json
import os
import shutil
import struct
import tempfile

import numpy as np
import pytest

from curvine_b200 import fs as F
from curvine_b200 import safetensors as ST

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden():
    spec = importlib.util.spec_from_file_location("make_safetensors_golden", os.path.join(ROOT, "tests", "golden", "make_safetensors_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


G = _golden()
RECORD = G.load()["checkpoints"]
CKS = sorted(RECORD)


def official_file(ck):
    """the rebuilt bytes of checkpoint `ck`, checked against the SHA-256 of the file safetensors.torch.save wrote"""
    blob = G.rebuild(ck, RECORD[ck]["header"])
    assert len(blob) == RECORD[ck]["size"] and hashlib.sha256(blob).hexdigest() == RECORD[ck]["sha256"], ck
    return blob


def _official():
    try:
        import safetensors
        return safetensors
    except ImportError:
        return None


def parse(blob):
    return ST.parse_header(lambda o, n: blob[o:o + n], len(blob))


def _header(blob):
    (n,) = struct.unpack("<Q", blob[:8])
    return {k: v for k, v in json.loads(blob[8:8 + n]).items() if k != "__metadata__"}


@pytest.mark.parametrize("ck", CKS)
def test_rebuilt_files_are_the_official_writers(ck):
    official_file(ck)
    assert RECORD[ck]["spec"] == json.loads(json.dumps(G.CHECKPOINTS[ck])), "the generator's spec changed: regenerate the record"


def test_the_installed_official_writer_reproduces_the_record():
    if _official() is None:
        pytest.skip("the safetensors package is not installed")
    with open(G.JSON) as f:
        assert f.read() == G.generate()


@pytest.mark.parametrize("ck", CKS)
def test_parse_header_reads_official_files_as_their_header_states(ck, tmp_path):
    import torch
    blob = official_file(ck)
    start, ents = parse(blob)
    hdr = _header(blob)
    assert start == 8 + struct.unpack("<Q", blob[:8])[0] and start % 8 == 0
    assert set(ents) == set(hdr)
    table = ST.dtypes()
    for name, e in hdr.items():
        dt, shape, b, end = ents[name]
        assert dt == table.get(e["dtype"], e["dtype"]) and list(shape) == e["shape"] and [b, end] == e["data_offsets"], name
        assert isinstance(dt, torch.dtype) == (e["dtype"] not in ("F4", "F6_E2M3", "F6_E3M2")), name
    assert {n for n, (dt, *_) in ents.items() if isinstance(dt, str)} == {n for n, e in hdr.items() if e["dtype"] == "F4"}
    st = _official()
    if st is None:
        return
    p = tmp_path / "m.safetensors"
    p.write_bytes(blob)
    from safetensors import safe_open
    with safe_open(str(p), framework="numpy") as f:
        assert set(f.keys()) == set(ents)
        for name in f.keys():
            sl = f.get_slice(name)
            assert sl.get_dtype() == hdr[name]["dtype"] and tuple(sl.get_shape()) == ents[name][1], name
    for name, t in st.deserialize(blob):  # and the bytes the official reader hands out are the ones at the parsed offsets
        _, _, b, end = ents[name]
        assert bytes(t["data"]) == blob[start + b:start + end], name


def _one(dt, shape, n):
    h = json.dumps({"a": {"dtype": dt, "shape": shape, "data_offsets": [0, n]}}).encode()
    h += b" " * (-(8 + len(h)) % 8)
    return struct.pack("<Q", len(h)) + h + bytes(n)


def _official_accepts(blob):
    st = _official()
    if st is None:
        return None
    try:
        st.deserialize(blob)
        return True
    except Exception:
        return False


# every dtype name of the format and its width in bits, as the official reader lists them
WIDTH = {"BOOL": 8, "F4": 4, "F6_E2M3": 6, "F6_E3M2": 6, "U8": 8, "I8": 8, "F8_E5M2": 8, "F8_E4M3": 8, "F8_E8M0": 8, "I16": 16, "U16": 16,
         "F16": 16, "BF16": 16, "I32": 32, "U32": 32, "F32": 32, "C64": 64, "F64": 64, "I64": 64, "U64": 64}


@pytest.mark.parametrize("dt", sorted(WIDTH))
def test_every_dtype_name_of_the_format_parses_with_its_width(dt):
    bits = WIDTH[dt]
    for shape in ([8], [2, 4], [], [0, 3]):
        n = 1
        for d in shape:
            n *= d
        if n * bits % 8:
            continue
        blob = _one(dt, shape, n * bits // 8)
        assert parse(blob)[1]["a"][:2] == (ST.dtypes().get(dt, dt), tuple(shape))
        assert _official_accepts(blob) in (None, True), (dt, shape)
    for extra in (-1, 1):  # one byte short, one byte over
        blob = _one(dt, [8], bits + extra)
        with pytest.raises(ST.SafetensorsError, match="needs %d bytes" % bits):
            parse(blob)
        assert _official_accepts(blob) in (None, False), dt


# sub-byte tensors: what the format's own reader decides, which this parser must match
@pytest.mark.parametrize("dt,shape,n,ok", [
    ("F6_E2M3", [4], 3, True), ("F6_E3M2", [2, 4], 6, True), ("F4", [4], 2, True), ("F4", [2, 3], 3, True), ("F4", [0], 0, True),
    ("F4", [3], 2, False), ("F4", [3], 1, False), ("F6_E3M2", [3], 3, False), ("F6_E2M3", [1], 1, False), ("F4", [4], 3, False),
    ("F6_E2M3", [4], 4, False), ("F8_E8M0", [3], 3, True), ("C64", [2], 16, True), ("C64", [2], 8, False),
])
def test_sub_byte_sizes_are_decided_as_the_official_reader_decides(dt, shape, n, ok):
    blob = _one(dt, shape, n)
    if ok:
        assert parse(blob)[1]["a"][1] == tuple(shape)
    else:
        with pytest.raises(ST.SafetensorsError, match="byte boundary|needs"):
            parse(blob)
    assert _official_accepts(blob) in (None, ok)


def test_unknown_and_malformed_dtype_names_are_rejected():
    for dt in ("F8_E4M3FNUZ", "C128", "U4", "f32", "", None, 4, ["F32"]):
        with pytest.raises(ST.SafetensorsError, match="unknown dtype"):
            parse(_one(dt, [1], 4))


@pytest.fixture(scope="module")
def fs_with_official_files():
    d = tempfile.mkdtemp(prefix="cvsf", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    w = F.MiniWorker(["[MEM]" + d + "/m"])
    fs = F.CurvineFileSystem(F.client_conf(short_circuit=False))
    for k, ck in enumerate(CKS):
        wr = fs.create("/sf/" + ck, 8300 + k, 64 << 10, w.port, chunk_size=32768)
        wr.write(official_file(ck))
        wr.complete()
    yield fs
    fs.close()
    w.stop()
    shutil.rmtree(d, ignore_errors=True)


def test_unloadable_tensors_are_listed_but_refused_before_anything_is_read(fs_with_official_files):
    import torch
    fs = fs_with_official_files
    hdr = ST.read_header(fs, "/sf/tiles_128x128")
    assert hdr["mx.f4"] == ("F4", (5, 6)) and hdr["mx.scales"] == (torch.float8_e8m0fnu, (4, 7)) and hdr["rope.c64"] == (torch.complex64, (3,))
    for names in (None, ["mx.f4"], ["norm.f32", "mx.f4"]):
        with pytest.raises(ValueError, match=r"mx\.f4: its dtype F4 has no torch dtype"):
            ST.load_file(fs, "/sf/tiles_128x128", device="cpu", names=names)
    with pytest.raises(ValueError, match=r"fp4: its dtype F4"):
        ST.load_file(fs, "/sf/tiles_64x48", device="cpu")
    start, ents = parse(official_file("tiles_128x128"))
    # F8_E8M0 is a float8 type: dtype= and scales= refuse it like the others; complex64 stays as stored under dtype=
    with pytest.raises(ValueError, match=r"mx\.scales: torch\.float8_e8m0fnu tensors are not converted"):
        ST.plan_ranges(start, ents, ["mx.scales"], dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="must be F8_E4M3 or F8_E5M2"):
        ST.plan_ranges(start, ents, ["mx.scales"], dtype=torch.bfloat16, scales={"mx.scales": "q.weight_scale"})
    with pytest.raises(ValueError, match="must be F32, F16 or BF16"):
        ST.plan_ranges(start, ents, ["q.weight"], dtype=torch.bfloat16, scales={"q.weight": "mx.scales"})
    (_, dt, shape, rng), = ST.plan_ranges(start, ents, ["rope.c64"], dtype=torch.float16)
    assert dt == torch.complex64 and shape == (3,) and rng[5:] == (torch.complex64, torch.complex64)
    (_, dt, _, _), = ST.plan_ranges(start, ents, ["mx.scales"])
    assert dt == torch.float8_e8m0fnu


def _rank_slices(shape, world):
    """(dim, start, stop) of every rank of `world` on dims 0, 1 and -1 that the tensor has: uneven and empty shards included"""
    out = []
    for dim in (0, 1, -1):
        if -len(shape) <= dim < len(shape):
            size = shape[dim]
            out += [(dim, r * size // world, (r + 1) * size // world) for r in range(world)]
    return out


def _read_bytes(rng):
    """the file bytes a range (file_off, row_len, rows, file_pitch, ...) reads, in destination order"""
    off, L, R, P = rng[:4]
    return (off + np.arange(R, dtype=np.int64)[:, None] * P + np.arange(L, dtype=np.int64)[None, :]).ravel()


@pytest.mark.parametrize("ck", CKS)
def test_plan_ranges_reads_what_a_numpy_slice_selects(ck):
    """every loadable tensor, whole and for every rank of worlds 2, 3 and 8 on dims 0, 1 and -1, as stored, cast and dequantized:
    the planned rows read exactly the bytes numpy's slice of the element grid names, in order; the destination is the result packed"""
    import torch
    blob = official_file(ck)
    start, ents = parse(blob)
    spec = RECORD[ck]["spec"]
    scales, block = spec["scales"], tuple(spec["scale_block"])
    names = [n for n, (dt, *_) in ents.items() if not isinstance(dt, str)]
    for dtype, sc in ((None, None), (torch.bfloat16, None), (torch.float32, scales)):
        refused = () if dtype is None else (torch.float8_e8m0fnu,) if sc else (torch.float8_e4m3fn, torch.float8_e5m2, torch.float8_e8m0fnu)
        sel = [n for n in names if ents[n][0] not in refused]
        for world in (1, 2, 3, 8):
            cases = [{}] if world == 1 else [{n: s} for n in sel for s in _rank_slices(ents[n][1], world)]
            for sl in cases:
                plan = ST.plan_ranges(start, ents, sel, sl, dtype, sc, block if sc else None)
                assert [p[0] for p in plan] == sel
                for name, dt, shape, rng in plan:
                    stored, full, b, _ = ents[name]
                    isz = stored.itemsize
                    grid = np.arange(int(np.prod(full, dtype=np.int64)), dtype=np.int64).reshape(full)
                    if name in sl:
                        d, a, z = sl[name]
                        grid = np.take(grid, np.arange(a, z), axis=d)
                    assert shape == grid.shape, (name, sl)
                    want = (start + b + grid.ravel()[:, None] * isz + np.arange(isz)[None, :]).ravel()
                    got = _read_bytes(rng) if rng is not None else np.zeros(0, dtype=np.int64)
                    assert np.array_equal(got, want), (name, sl, dtype)
                    if rng is None:
                        continue
                    res = dt.itemsize
                    assert rng[2] == 1 or rng[4] == rng[1] // isz * res, (name, sl)  # rows land back to back
                    if sc is not None and name in sc:
                        assert dt == dtype and rng[7][0] == sc[name] and rng[7][6] == int(grid.ravel()[0]), (name, sl)
                    elif dtype is not None and stored in (torch.float32, torch.float16, torch.bfloat16):
                        assert dt == dtype and rng[5:7] == (stored, dtype)
                    else:
                        assert dt == stored
