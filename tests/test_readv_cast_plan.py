"""Cast reads without a GPU: the plan cv_readv_cast_device executes (cv_readv_cast_plan) against a Python restatement over plain, strided
and converting ranges, the rule that no block a conversion touches is direct, the destination offsets of converting spans, the
equivalence of src == dst with the strided plan, rejection of malformed converting ranges, and what safetensors.load_file(dtype=...)
validates and builds."""
import ctypes
import os
import shutil
import tempfile

import numpy as np
import pytest

from curvine_b200 import _lib, fs as F
from curvine_b200 import safetensors as ST
from test_readv_strided_plan import model_strided_plan

BS = 4096


def _torch():
    import torch
    return torch


def model_cast_plan(ranges, block_lens):
    """ranges: (file_off, row_len, rows, file_pitch, dst_pitch, src itemsize, dst itemsize, converts) -> the strided plan, with every block
    a converting range touches not direct"""
    spans, nb, fetch = model_strided_plan([r[:5] for r in ranges], block_lens)
    cast_blocks = {s[0] for s in spans if ranges[s[4]][7]}
    return [s[:5] + (s[5] and s[0] not in cast_blocks,) for s in spans], nb, fetch


def dst_map(spans, ranges, block_lens):
    """destination element -> file offset of its source element, for every converting span: the in-row offset scaled by
    dst size / src size, the row offset dst_pitch apart"""
    starts = np.concatenate([[0], np.cumsum(block_lens)]).tolist()
    m = {}
    for b, bo, ln, rows, ri, _ in spans:
        off, L, R, P, dp, ss, ds, conv = ranges[ri]
        if not conv:
            continue
        for k in range(rows):
            f0 = starts[b] + bo + k * P
            rel = f0 - off
            row, col = (rel // P, rel % P) if R > 1 else (0, rel)
            for e in range(ln // ss):
                m[(ri, row * dp + (col // ss + e) * ds)] = f0 + e * ss
    return m


def random_cast(rng, n, max_ranges):
    """non-overlapping extents in random order: plain byte ranges, strided ranges, converting ranges (all six conversions) at element
    alignment, some empty"""
    torch = _torch()
    fl = [torch.float32, torch.float16, torch.bfloat16]
    cuts = sorted(set(int(x) for x in rng.integers(0, n + 1, size=2 * int(rng.integers(1, max_ranges + 1)))))
    out = []
    for a, b in zip(cuts[::2], cuts[1::2]):
        kind = rng.random()
        if kind < 0.3:
            src = dst = torch.uint8
        elif kind < 0.4:
            src = dst = fl[int(rng.integers(0, 3))]
        else:
            src, dst = [fl[int(i)] for i in rng.choice(3, 2, replace=False)]
        ss, ds = src.itemsize, dst.itemsize
        a = (a + ss - 1) // ss * ss
        ext = (b - a) // ss * ss
        if ext <= 0:
            continue
        L = ss * int(rng.integers(1, min(ext, 3 * BS) // ss + 1))
        if ext == L or rng.random() < 0.3:
            out.append((a, L, 1, 0, 0, src, dst))
            continue
        P = ss * int(rng.integers(L // ss, ext // ss + 1))
        R = 1 + (ext - L) // P
        out.append((a, L, R, P, L // ss * ds + ds * int(rng.integers(0, 5)), src, dst))
    rng.shuffle(out)
    return out


@pytest.fixture(scope="module")
def files():
    d = tempfile.mkdtemp(prefix="cvcp", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    w = F.MiniWorker(["[MEM]" + d + "/m"])
    mans = [w.create_file("/cp/a", 9950, 40 * BS - 1000, BS, threads=2), w.create_file("/cp/odd", 9951, 10 * 4098, 4098, threads=2)]
    fs = F.CurvineFileSystem(F.client_conf())
    for m in mans:
        fs.load_namespace(m)
    yield fs
    fs.close()
    w.stop()
    shutil.rmtree(d, ignore_errors=True)


def _model_ranges(rs):
    return [(o, L, R, P, dp, s.itemsize, d.itemsize, s != d) for o, L, R, P, dp, s, d in rs]


def test_cast_plan_matches_the_restatement(files):
    fs = files
    n = 40 * BS - 1000
    lens = [min(BS, n - i) for i in range(0, n, BS)]
    rng = np.random.default_rng(31)
    torch = _torch()
    edge = [
        [(0, n, 1, 0, 0, torch.float32, torch.bfloat16)],                               # the whole file: not one block direct
        [(BS - 4, 12, 6, 3 * BS + 8, 8, torch.float32, torch.float16)],                  # every row crosses a block edge
        [(2, 2 * BS + 300, 4, 3 * BS, 4 * BS + 600, torch.bfloat16, torch.float32)],     # whole blocks inside rows, 2x wider in HBM
        [(0, 3 * BS, 1, 0, 0, torch.uint8, torch.uint8), (3 * BS, BS, 1, 0, 0, torch.float16, torch.bfloat16)],  # direct next to converted
        [(0, 8, 0, 16, 4, torch.float32, torch.bfloat16), (40, 0, 3, 8, 4, torch.float16, torch.float32)],       # empty ranges touch nothing
    ]
    sets = edge + [random_cast(rng, n, 10) for _ in range(60)]
    with fs.open("/cp/a") as r:
        for rs in sets:
            got = r.readv_cast_plan([(o, L, R, P, 0, dp, s, d) for o, L, R, P, dp, s, d in rs])
            model = _model_ranges(rs)
            assert got == model_cast_plan(model, lens), rs
            spans = got[0]
            for b in {s[0] for s in spans if model[s[4]][7]}:
                assert not any(s[5] for s in spans if s[0] == b), (rs, b)  # no block a conversion touches is direct
            # every destination element of every converting range is delivered exactly once, from its own source element
            m = dst_map(spans, model, lens)
            want = {}
            for i, (o, L, R, P, dp, ss, ds, conv) in enumerate(model):
                for k in range(R if conv and L else 0):
                    for e in range(L // ss):
                        want[(i, k * dp + e * ds)] = o + k * P + e * ss
            assert m == want, rs
        assert r.pos() == 0


def test_same_dtype_plans_exactly_like_the_strided_plan(files):
    fs = files
    torch = _torch()
    n = 40 * BS - 1000
    rng = np.random.default_rng(8)
    with fs.open("/cp/a") as r:
        for _ in range(30):
            rs = random_cast(rng, n, 8)
            for dt in (torch.float32, torch.bfloat16, torch.uint8):
                same = [(o, L, R, P, 0, max(dp, L), dt, dt) for o, L, R, P, dp, _, _ in rs]
                assert r.readv_cast_plan(same) == r.readv_strided_plan([x[:6] for x in same]), same


def _raw_plan(r, rng_):
    """cv_readv_cast_plan on one CvCastRange of raw dtype codes"""
    arr = (_lib.CvCastRange * 2)()
    a = arr[1]
    a.file_off, a.row_len, a.rows, a.file_pitch, a.d_dst, a.dst_pitch, a.src_dtype, a.dst_dtype = rng_
    arr[0].file_off, arr[0].row_len, arr[0].rows = 0, 4, 1  # range 0 is fine: the error must name range 1
    return _lib.lib().cv_readv_cast_plan(r._h, arr, 2, None, None, None, None, None, None, 0, None, None, None)


F32, F16, BF16, NONE = _lib.DTYPE_F32, _lib.DTYPE_F16, _lib.DTYPE_BF16, _lib.DTYPE_NONE


@pytest.mark.parametrize("rng_,what", [
    ((64, 8, 1, 0, 0, 0, 7, 7), "unknown dtype code 7"),
    ((64, 8, 1, 0, 0, 0, F32, -1), "unknown dtype code -1"),
    ((64, 8, 1, 0, 0, 0, NONE, F32), "conversions are between F32, F16 and BF16 only"),
    ((64, 8, 1, 0, 0, 0, BF16, NONE), "conversions are between F32, F16 and BF16 only"),
    ((66, 8, 1, 0, 0, 0, F32, BF16), "multiples of the source element size"),
    ((64, 6, 1, 0, 0, 0, F32, BF16), "multiples of the source element size"),
    ((64, 8, 2, 10, 0, 8, F32, F16), "multiples of the source element size"),
    ((64, 3, 1, 0, 0, 0, F16, F32), "multiples of the source element size"),
    ((64, 8, 1, 0, 2, 0, F16, F32), "multiples of the destination element size"),
    ((64, 8, 1, 0, 1, 0, F32, BF16), "multiples of the destination element size"),
    ((64, 8, 2, 8, 0, 10, BF16, F32), "multiples of the destination element size"),
    ((64, 8, 2, 8, 0, 12, BF16, F32), "pitch shorter"),                        # a float32 row of 4 elements is 16 bytes
    ((64, 16, 2, 16, 0, 6, F32, BF16), "pitch shorter"),
    ((64, 8, 3, 8, 0, 1 << 62, BF16, F32), "overflows"),
    ((40 * BS - 1008, 12, 1, 0, 0, 0, F32, BF16), "outside the file"),
])
def test_malformed_cast_ranges_are_errors_that_name_the_range(files, rng_, what):
    fs = files
    with fs.open("/cp/a") as r:
        assert _raw_plan(r, rng_) == -10000
        msg = _lib.lib().cv_last_error().decode()
        assert "range 1" in msg and what in msg, msg
        assert _raw_plan(r, (64, 8, 2, 8, 0, 4, F32, BF16)) == 0  # a row of 2 float32 -> 4 bytes of bfloat16: fine, reader still usable


def test_a_block_size_that_splits_elements_is_an_error(files):
    fs = files
    torch = _torch()
    with fs.open("/cp/odd") as r:  # 4098-byte blocks: whole bfloat16 elements, not whole float32 ones
        with pytest.raises(F.FsError, match=r"range 0\b.*block size 4098"):
            r.readv_cast_plan([(0, 40, 1, 0, 0, 0, torch.float32, torch.bfloat16)])
        spans, nb, _ = r.readv_cast_plan([(4000, 400, 1, 0, 0, 0, torch.bfloat16, torch.float32)])
        assert nb == 2 and [s[2] for s in spans] == [98, 302]
        with pytest.raises(ValueError, match="range 0"):
            r.readv_cast_plan([(0, 40, 1, 0, 0, 0, torch.int32, torch.float32)])  # integer conversions are refused before the call


# ---- safetensors.load_file(dtype=...): validation and range construction (safetensors.plan_ranges)

def _entries():
    torch = _torch()
    ents = {"w": (torch.float32, (6, 8), 0, 192), "h": (torch.float16, (8,), 192, 208), "t": (torch.int8, (2, 3, 4), 208, 232),
            "s": (torch.float64, (), 232, 240), "z": (torch.bfloat16, (0, 4), 240, 240), "b": (torch.bfloat16, (4, 2), 240, 256)}
    return 1000, ents


def test_dtype_ranges_convert_floats_and_keep_the_rest():
    torch = _torch()
    start, ents = _entries()
    names = ["w", "h", "t", "z", "b"]
    got = {n: (dt, shape, rng) for n, dt, shape, rng in ST.plan_ranges(start, ents, names, dtype=torch.bfloat16)}
    assert got["w"] == (torch.bfloat16, (6, 8), (1000, 192, 1, 0, 0, torch.float32, torch.bfloat16))
    assert got["h"] == (torch.bfloat16, (8,), (1192, 16, 1, 0, 0, torch.float16, torch.bfloat16))
    assert got["t"] == (torch.int8, (2, 3, 4), (1208, 24, 1, 0, 0, torch.int8, torch.int8))       # integers as stored
    assert got["z"] == (torch.bfloat16, (0, 4), None) and got["b"][2][5:] == (torch.bfloat16, torch.bfloat16)
    # slices: the file side in stored bytes, dst_pitch in result bytes
    got = {n: (shape, rng) for n, _, shape, rng in ST.plan_ranges(start, ents, names, {"w": (1, 2, 6), "t": (-1, 1, 3)}, dtype=torch.float16)}
    assert got["w"] == ((6, 4), (1000 + 2 * 4, 4 * 4, 6, 8 * 4, 4 * 2, torch.float32, torch.float16))
    assert got["t"] == ((2, 3, 2), (1208 + 1, 2, 6, 4, 2, torch.int8, torch.int8))
    got = {n: rng for n, _, _, rng in ST.plan_ranges(start, ents, ["h"], {"h": (0, 2, 5)}, dtype=torch.float32)}
    assert got == {"h": (1192 + 4, 6, 1, 16, 12, torch.float16, torch.float32)}
    # dtype=None: the ranges of readv_strided_device, unchanged
    assert ST.plan_ranges(start, ents, ["w"])[0][3] == (1000, 192, 1, 0, 0)


@pytest.mark.parametrize("selected,dtype,what", [
    (["w", "s"], "bfloat16", "s: torch.float64"),
    (["w"], "float64", "convert to float32, float16 or bfloat16 only"),
    (["w"], "int32", "convert to float32, float16 or bfloat16 only"),
])
def test_tensors_dtype_cannot_convert_are_rejected(selected, dtype, what):
    start, ents = _entries()
    with pytest.raises(ValueError, match=what):
        ST.plan_ranges(start, ents, selected, dtype=getattr(_torch(), dtype))


def test_float8_and_misaligned_tensors_are_rejected_by_name():
    torch = _torch()
    start, ents = _entries()
    ents = dict(ents, f8=(torch.float8_e4m3fn, (4,), 256, 260))
    with pytest.raises(ValueError, match="f8: torch.float8_e4m3fn"):
        ST.plan_ranges(start, ents, ["w", "f8"], dtype=torch.float16)
    with pytest.raises(ValueError, match="w: data offset 1002"):
        ST.plan_ranges(1002, ents, ["t", "w"], dtype=torch.float16)
    assert ST.plan_ranges(1001, ents, ["t"], dtype=torch.float16)[0][3][0] == 1209  # an int8 tensor is not converted: any offset
    assert ST.plan_ranges(1002, ents, ["w"], dtype=torch.float32)[0][3][5:] == (torch.float32, torch.float32)  # nor one already float32


class _FakeReader:
    """Reader stand-in: serves a safetensors blob from memory and records the vectored read instead of doing it"""
    def __init__(self, blob):
        self.blob, self.pos, self.calls = blob, 0, []

    def len(self):
        return len(self.blob)

    def seek(self, p):
        self.pos = p

    def read_full(self, n):
        return self.blob[self.pos:self.pos + n]

    def readv_strided_device(self, ranges, stream=0):
        self.calls.append(("strided", ranges))
        return sum(r[1] * r[2] for r in ranges)

    def readv_cast_device(self, ranges, stream=0):
        self.calls.append(("cast", ranges))
        return 0

    def verify(self):
        return 0, 0, 0

    def complete(self):
        pass


def test_load_file_dtype_validates_before_reading_and_issues_one_call(monkeypatch):
    torch = _torch()
    from test_readv_plan import write_safetensors
    blob = write_safetensors([("w", "F32", (6, 8), bytes(192)), ("i", "I32", (2,), bytes(8)), ("d", "F64", (1,), bytes(8))], pad_to=8)
    rd = _FakeReader(blob)
    fake_fs = type("FS", (), {"open": lambda self, p: rd})()
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: type("S", (), {"cuda_stream": 0})())
    allocs = []
    real_empty = torch.empty
    monkeypatch.setattr(torch, "empty", lambda *a, **k: allocs.append(a) or real_empty(*a, **{**k, "device": "cpu"}))
    for kw in (dict(dtype=torch.bfloat16), dict(dtype=torch.int8, names=["w"])):
        with pytest.raises(ValueError):
            ST.load_file(fake_fs, "/x", device="cpu", **kw)
    assert not allocs and not rd.calls  # nothing allocated, nothing read
    out = ST.load_file(fake_fs, "/x", device="cpu", names=["w", "i"], slices={"w": (1, 4, 8)}, dtype=torch.bfloat16)
    assert out["w"].dtype == torch.bfloat16 and tuple(out["w"].shape) == (6, 4) and out["i"].dtype == torch.int32
    (kind, (w, i)), start = rd.calls[0], len(blob) - 208
    assert len(rd.calls) == 1 and kind == "cast"
    assert w[:4] == (start + 16, 16, 6, 32) and w[5:] == (8, torch.float32, torch.bfloat16)
    assert i[:4] == (start + 192, 8, 1, 0) and i[6:] == (torch.int32, torch.int32)
    ST.load_file(fake_fs, "/x", device="cpu", names=["w"])  # dtype=None: the strided call, as before
    assert rd.calls[-1][0] == "strided" and rd.calls[-1][1][0] == (start, 192, 1, 0, rd.calls[-1][1][0][4], 0)
