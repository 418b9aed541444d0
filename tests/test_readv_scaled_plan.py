"""FP8 loads without a GPU: the scale geometry safetensors.plan_ranges(scales=, scale_block=) hands to Reader.readv_scaled_device, checked
element by element against a restatement of the scale rule on the full tensor (per-tensor, per-row and block scales, edge tiles, dim-0
and dim-1 slices), every ValueError load_file(scales=...) raises, and the calls load_file makes with and without scales."""
import numpy as np
import pytest

from curvine_b200 import safetensors as ST
from test_readv_cast_plan import _FakeReader


def _torch():
    import torch
    return torch


def _ents(specs, start=1000):
    """specs: [(name, torch dtype, shape)] -> (data_start, entries) laid out back to back"""
    ents, at = {}, 0
    for name, dt, shape in specs:
        n = int(np.prod(shape)) * dt.itemsize
        ents[name] = (dt, tuple(shape), at, at + n)
        at += n
    return start, ents


def _scale_index_by_kernel_rule(rng, row_elems):
    """for every element of the range (rows of row_elems elements): the scale element the kernel multiplies it by"""
    _, _, rows, file_pitch, _, _, _, scale = rng
    _, scale_rows, scale_cols, br, bc, cols, first = scale
    out = []
    for k in range(rows):
        for e in range(row_elems):
            v = first + k * file_pitch + e  # an F8 element is one byte
            i, j = divmod(v, cols)
            out.append((i // br) * scale_cols + j // bc)
    assert max(out) < scale_rows * scale_cols
    return out


def _scale_index_reference(shape, sshape, block, slc):
    """the same, from the definition: the sliced elements' positions in the full tensor, as (row, col) of its 2-D view"""
    full = np.arange(int(np.prod(shape))).reshape(shape)
    if slc is not None:
        dim, a, b = slc
        full = np.take(full, range(a, b), axis=dim)
    cols = shape[-1]
    out = []
    for idx in full.reshape(-1):
        i, j = divmod(int(idx), cols)
        if int(np.prod(sshape)) == 1:
            out.append(0)
        elif tuple(sshape) == (shape[0], 1):
            out.append(i)  # per row
        else:
            out.append((i // block[0]) * sshape[1] + j // block[1])
    return out


CASES = [
    # weight shape, scale shape, scale_block, slice
    ((6, 40), (1,), None, None),                     # per tensor
    ((2, 3, 8), (), None, None),                     # per tensor, 3-D weight, 0-d scale
    ((6, 40), (6, 1), None, None),                   # per row
    ((6, 40), (6, 1), None, (1, 5, 29)),             # per row, dim-1 slice
    ((300, 260), (3, 3), (128, 128), None),          # 128x128 blocks, partial edge tiles in both dims
    ((300, 260), (3, 3), (128, 128), (0, 100, 300)),  # dim-0 slice across a tile edge
    ((300, 260), (3, 3), (128, 128), (1, 120, 260)),  # dim-1 slice across a tile edge
    ((37, 13), (10, 3), (4, 5), None),               # small tiles, C not a multiple of 8
    ((37, 13), (10, 3), (4, 5), (1, 3, 11)),
    ((37, 13), (10, 3), (4, 5), (0, 7, 30)),
    ((37, 13), (37, 1), (4, 5), (1, 2, 9)),          # (R, 1) is per row even when scale_block is given
]


@pytest.mark.parametrize("shape,sshape,block,slc", CASES)
def test_scale_geometry_matches_the_rule_for_every_element(shape, sshape, block, slc):
    torch = _torch()
    start, ents = _ents([("pad", torch.int8, (4,)), ("w_scale_inv", torch.float32, sshape), ("b", torch.bfloat16, (5,)),
                         ("w", torch.float8_e4m3fn, shape)])  # the weight last: its size may be odd
    plan = ST.plan_ranges(start, ents, ["w", "b", "w_scale_inv"], {"w": slc} if slc else None, torch.bfloat16, {"w": "w_scale_inv"}, block)
    got = {name: (dt, res, rng) for name, dt, res, rng in plan}
    dt, res, rng = got["w"]
    assert dt == torch.bfloat16 and rng[5:7] == (torch.float8_e4m3fn, torch.bfloat16) and rng[7][0] == "w_scale_inv"
    row_elems = rng[1]
    assert rng[2] * row_elems == int(np.prod(res))
    assert _scale_index_by_kernel_rule(rng, row_elems) == _scale_index_reference(shape, sshape, block, slc)
    # the other tensors: what plan_ranges(dtype=...) gives them, with no scale
    plain = {name: r for name, _, _, r in ST.plan_ranges(start, ents, ["b", "w_scale_inv"], None, torch.bfloat16)}
    assert got["b"][2] == plain["b"] + (None,) and got["w_scale_inv"][2] == plain["w_scale_inv"] + (None,)


def test_e5m2_weights_and_f16_bf16_scales_are_accepted():
    torch = _torch()
    start, ents = _ents([("w", torch.float8_e5m2, (4, 8)), ("s", torch.float16, (4, 1)), ("v", torch.float8_e4m3fn, (8,)), ("t", torch.bfloat16, (1, 1))])
    got = {n: r for n, _, _, r in ST.plan_ranges(start, ents, ["w", "v"], dtype=torch.float32, scales={"w": "s", "v": "t"})}
    assert got["w"][5:] == (torch.float8_e5m2, torch.float32, ("s", 4, 1, 1, 8, 8, 0))
    assert got["v"][5:] == (torch.float8_e4m3fn, torch.float32, ("t", 1, 1, 1, 8, 8, 0))


def _bad_entries():
    torch = _torch()
    return _ents([("w", torch.float8_e4m3fn, (6, 40)), ("w3", torch.float8_e4m3fn, (2, 3, 4)), ("s", torch.float32, (6, 1)),
                  ("sb", torch.float32, (2, 3)), ("si", torch.int32, (1,)), ("h", torch.float16, (6, 40)), ("f8", torch.float8_e5m2, (4,)),
                  ("s1", torch.float32, (1,))])


@pytest.mark.parametrize("kw,what", [
    (dict(scales={"w": "s"}, dtype=None), "without dtype"),
    (dict(scales={"w": "nope"}), "w: its scale nope is not in the file"),
    (dict(scales={"w": "s", "s": "s1"}), "w: its scale s is itself a weight"),
    (dict(scales={"w": "w"}), "w: its scale w is itself a weight"),
    (dict(scales={"h": "s"}), r"h \(scale s\): a scaled weight must be F8_E4M3 or F8_E5M2"),
    (dict(scales={"w": "si"}), "w: its scale si must be F32, F16 or BF16"),
    (dict(scales={"w": "sb"}), r"w \(6, 40\): its scale sb has shape \(2, 3\)"),  # blocks need scale_block
    (dict(scales={"w": "sb"}, scale_block=(4, 32)), r"its scale sb has shape \(2, 3\)"),  # the blocks would be (2, 2)
    (dict(scales={"w3": "s"}), r"w3 \(2, 3, 4\): its scale s has shape \(6, 1\)"),  # per-row scales are for 2-D weights
    (dict(scales={"missing": "s"}), r"missing \(scale s\): the file holds no such weight"),
    (dict(scales={"w": "s"}, scale_block=(0, 128)), "scale_block"),
    (dict(scales={"w": "s"}, scale_block=(128,)), "scale_block"),
    (dict(scale_block=(128, 128)), "scale_block is given without scales"),
    (dict(scales={"w": "s"}, names=["w", "f8"]), "f8: torch.float8_e5m2"),  # an FP8 tensor without a scale keeps today's error
])
def test_scale_errors_name_the_weight_and_its_scale(kw, what):
    torch = _torch()
    start, ents = _bad_entries()
    kw = dict(kw)
    names = kw.pop("names", ["w", "w3"])
    dtype = kw.pop("dtype", torch.bfloat16)
    with pytest.raises(ValueError, match=what):
        ST.plan_ranges(start, ents, names, dtype=dtype, **kw)


class _ScaledFakeReader(_FakeReader):
    def readv_scaled_device(self, ranges, stream=0):
        self.calls.append(("scaled", ranges))
        return 0


def _fake(monkeypatch, blob):
    torch = _torch()
    rd = _ScaledFakeReader(blob)
    fake_fs = type("FS", (), {"open": lambda self, p: rd})()
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: type("S", (), {"cuda_stream": 0})())
    allocs = []
    real_empty = torch.empty
    monkeypatch.setattr(torch, "empty", lambda *a, **k: allocs.append(a) or real_empty(*a, **{**k, "device": "cpu"}))
    return rd, fake_fs, allocs


def test_load_file_scales_validates_before_reading_and_issues_two_calls(monkeypatch):
    torch = _torch()
    from test_readv_plan import write_safetensors
    blob = write_safetensors([("w", "F8_E4M3", (6, 40), bytes(240)), ("w_scale_inv", "F32", (1, 1), bytes(4)), ("i", "I32", (2,), bytes(8)),
                              ("r", "F8_E5M2", (6, 40), bytes(240)), ("r_s", "BF16", (6, 1), bytes(12))], pad_to=8)
    rd, fake_fs, allocs = _fake(monkeypatch, blob)
    for kw in (dict(scales={"w": "w_scale_inv"}),                                            # no dtype
               dict(scales={"w": "w_scale_inv"}, dtype=torch.bfloat16),                      # r is FP8 without a scale
               dict(scales={"w": "w_scale_inv", "r": "i"}, dtype=torch.bfloat16),            # an integer scale
               dict(scales={"w": "w_scale_inv", "r": "r_s"}, scale_block=(1,), dtype=torch.bfloat16)):
        with pytest.raises(ValueError):
            ST.load_file(fake_fs, "/x", device="cpu", **kw)
    assert not allocs and not rd.calls  # nothing allocated, nothing read
    start = len(blob) - 504
    out = ST.load_file(fake_fs, "/x", device="cpu", scales={"w": "w_scale_inv", "r": "r_s"}, slices={"r": (1, 8, 16)}, dtype=torch.float16)
    assert [k for k, _ in rd.calls] == ["strided", "scaled"]
    # 1: the scale tensors as stored, into temporaries
    (_, scl), (_, rs) = rd.calls
    assert [s[:4] for s in scl] == [(start + 240, 4, 1, 0), (start + 492, 12, 1, 0)]
    # 2: every selected tensor, the weights with their scales' temporaries
    w, s, i, r, r_s = rs
    assert w[:4] == (start, 240, 1, 0) and w[6:8] == (torch.float8_e4m3fn, torch.float16)
    assert w[8][0] == scl[0][4] and w[8][1:] == (torch.float32, 1, 1, 6, 40, 40, 0)
    assert r[:4] == (start + 252 + 8, 8, 6, 40) and r[8][0] == scl[1][4] and r[8][1:] == (torch.bfloat16, 6, 1, 1, 40, 40, 8)
    assert s[6:] == (torch.float32, torch.float16, None) and i[6:] == (torch.int32, torch.int32, None)
    assert r_s[6:] == (torch.bfloat16, torch.float16, None)
    assert out["w"].dtype == torch.float16 and tuple(out["r"].shape) == (6, 8) and out["w_scale_inv"].dtype == torch.float16
    assert out["i"].dtype == torch.int32
    # without scales: exactly the single call of before
    del rd.calls[:]
    ST.load_file(fake_fs, "/x", device="cpu", names=["i"], dtype=torch.float16)
    ST.load_file(fake_fs, "/x", device="cpu", names=["i"])
    assert [k for k, _ in rd.calls] == ["cast", "strided"]
