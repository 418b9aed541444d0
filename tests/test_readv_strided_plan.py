"""Strided vectored reads without a GPU: the plan cv_readv_strided_device executes (cv_readv_strided_plan) against a Python restatement,
its equivalence with the plan of the same rows as plain ranges, its size on a tensor-parallel slice, rejection of malformed strided
ranges, and the ranges safetensors.load_file(slices=...) builds."""
import ctypes
import os
import shutil
import tempfile

import numpy as np
import pytest

from curvine_b200 import _lib, fs as F
from curvine_b200 import safetensors as ST

BS = 4096


def model_strided_plan(ranges, block_lens):
    """-> (spans, n_blocks, fetch_bytes) as Reader.readv_strided_plan returns them, restated row by row: the pieces of one range inside
    one block are a clipped first row, a run of whole rows (one span), a clipped last row."""
    starts = np.concatenate([[0], np.cumsum(block_lens)]).tolist()
    spans = []
    for i in sorted((i for i, r in enumerate(ranges) if r[1] > 0 and r[2] > 0), key=lambda i: ranges[i][0]):
        off, L, R, P = ranges[i][:4]
        pieces = []  # (block, block_off, len, whole row)
        for k in range(R):
            p, end = off + k * P, off + k * P + L
            while p < end:
                b = next(b for b in range(len(block_lens)) if starts[b] <= p < starts[b + 1])
                take = min(end, starts[b + 1]) - p
                pieces.append((b, p - starts[b], take, take == L))
                p += take
        for b, bo, ln, whole in pieces:
            if whole and spans and spans[-1][5] and spans[-1][0] == b and spans[-1][4] == i:
                spans[-1][3] += 1
            else:
                spans.append([b, bo, ln, 1, i, whole])
    per_block = {}
    for s in spans:
        per_block.setdefault(s[0], []).append(s)
    out = [(s[0], s[1], s[2], s[3], s[4], len(per_block[s[0]]) == 1 and s[3] == 1 and s[1] == 0 and s[2] == block_lens[s[0]]) for s in spans]
    return out, len(per_block), sum(block_lens[b] for b in per_block)


def byte_map(spans, ranges, block_lens, strided=True):
    """file byte -> (range, destination offset) for every byte a plan delivers"""
    starts = np.concatenate([[0], np.cumsum(block_lens)]).tolist()
    m = {}
    for s in spans:
        b, bo, ln = s[0], s[1], s[2]
        rows, ri = (s[3], s[4]) if strided else (1, s[3])
        off, L, R, P, dp = ranges[ri]
        for k in range(rows):
            f0 = starts[b] + bo + k * P
            rel = f0 - off
            row, col = (rel // P, rel % P) if R > 1 else (0, rel)
            for x in range(ln):
                m[f0 + x] = (ri, row * dp + col + x)
    return m


def per_row(ranges):
    """the same rows as plain ranges -> (plain ranges, index of each plain range's strided range and row)"""
    plain, owner = [], []
    for i, (off, L, R, P, dp) in enumerate(ranges):
        for k in range(R if L else 0):
            plain.append((off + k * P, L, 0))
            owner.append((i, k))
    return plain, owner


def random_strided(rng, n, max_ranges):
    """Non-overlapping extents in random order; inside each, rows of a random length and pitch (some empty ranges)."""
    cuts = sorted(set(int(x) for x in rng.integers(0, n + 1, size=2 * int(rng.integers(1, max_ranges + 1)))))
    out = []
    for a, b in zip(cuts[::2], cuts[1::2]):
        ext = b - a
        if ext == 0 or rng.random() < 0.15:
            continue
        L = int(rng.integers(1, min(ext, 3 * BS) + 1))
        if ext == L:
            out.append((a, L, 1, L, L))
            continue
        P = int(rng.integers(L, ext + 1))
        R = 1 + (ext - L) // P
        out.append((a, L, R, P, L + int(rng.integers(0, 9))))
    out += [(int(rng.integers(0, n + 1)), 0, 3, 10, 10)] * int(rng.integers(0, 2))
    rng.shuffle(out)
    return out


@pytest.fixture(scope="module")
def files():
    d = tempfile.mkdtemp(prefix="cvsp", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    w = F.MiniWorker(["[MEM]" + d + "/m"])
    specs = {"/sp/a": (40 * BS - 999, 0), "/sp/holes": (23 * BS + 5, 3)}
    mans = [w.create_file(p, 9700 + k, n, BS, mode=2 if he else 0, hole_every=he, threads=2) for k, (p, (n, he)) in enumerate(specs.items())]
    # a [8192, 28672] bf16 tensor in 4 MiB blocks: every block a hole, so only the block table exists (the plan needs nothing else)
    mans.append(w.create_file("/sp/big", 9709, 8192 * 28672 * 2, 4 << 20, mode=2, hole_every=1, threads=2))
    fs = F.CurvineFileSystem(F.client_conf())
    for m in mans:
        fs.load_namespace(m)
    yield fs, {p: n for p, (n, _) in specs.items()}
    fs.close()
    w.stop()
    shutil.rmtree(d, ignore_errors=True)


def _edge_sets(n):
    return [
        [(BS - 5, 10, 6, 3 * BS + 7, 10)],              # every row crosses a block edge
        [(3, 1, 200, 97, 1)],                           # row_len = 1
        [(100, 2 * BS + 300, 4, 3 * BS, 2 * BS + 301)],  # rows longer than two blocks: whole blocks inside one row
        [(BS - 1, 64, 300, 64, 64)],                   # file_pitch = row_len: the rows are back to back
        [(17, 100, 5, 7 * BS + 3, 128)],                # sparse rows, several blocks apart: the blocks between are not touched
        [(0, 10, 0, 20, 10), (50, 0, 9, 20, 0)],        # rows = 0 and row_len = 0 touch nothing
        [(0, 8, 3, 16, 8), (40, 8, 1, 0, 8), (60, 1, 1, 1, 1)],  # plain ranges right behind a strided one
        [(0, n, 1, 0, 0)],                              # the whole file as one row: every block direct
        [],
    ]


def test_strided_plan_matches_the_restatement_and_the_per_row_plan(files):
    fs, sizes = files
    rng = np.random.default_rng(23)
    for path, n in sizes.items():
        lens = [min(BS, n - i) for i in range(0, n, BS)]
        sets = [[r for r in rs if r[0] + (r[2] - 1) * r[3] + r[1] <= n] for rs in _edge_sets(n)] + [random_strided(rng, n, 10) for _ in range(40)]
        with fs.open(path) as r:
            for rs in sets:
                got = r.readv_strided_plan([(o, L, R, P, 0, dp) for o, L, R, P, dp in rs])
                assert got == model_strided_plan(rs, lens), (path, rs)
                spans, nb, fetch = got
                assert sum(s[2] * s[3] for s in spans) == sum(L * R for _, L, R, _, _ in rs)
                # the same rows as plain ranges: same blocks, same fetch, same direct blocks, same file byte -> destination byte map
                plain, owner = per_row(rs)
                pspans, pnb, pfetch = r.readv_plan(plain)
                assert (nb, fetch) == (pnb, pfetch), rs
                assert {s[0] for s in spans if s[5]} == {s[0] for s in pspans if s[4]}
                want = {}
                for s in pspans:
                    i, k = owner[s[3]]
                    off, L, R, P, dp = rs[i]
                    f0 = sum(lens[:s[0]]) + s[1]
                    for x in range(s[2]):
                        want[f0 + x] = (i, k * dp + (f0 - off - k * P) + x)
                assert byte_map(spans, rs, lens) == want, rs
                # O(ranges + touched blocks): at most three spans for every (range, touched block) pair
                assert len(spans) <= 3 * len({(s[0], s[4]) for s in spans})
            assert r.pos() == 0


def test_sparse_rows_fetch_only_their_blocks(files):
    fs, sizes = files
    with fs.open("/sp/a") as r:
        spans, nb, fetch = r.readv_strided_plan([(17, 100, 5, 7 * BS + 3, 0, 100)])
        assert sorted({s[0] for s in spans}) == [0, 7, 14, 21, 28] and nb == 5 and fetch == 5 * BS


def test_a_tensor_parallel_slice_plans_in_spans_not_rows(files):
    """rank r of 8 of a [8192, 28672] bf16 tensor sliced on dim 1: 8192 rows of 7 KiB, 56 KiB apart, in 4 MiB blocks"""
    fs, _ = files
    rows, cols, world = 8192, 28672, 8
    row_len, pitch = cols // world * 2, cols * 2
    with fs.open("/sp/big") as r:
        for rank in (0, 3, 7):
            spans, nb, fetch = r.readv_strided_plan([(rank * row_len, row_len, rows, pitch, 0, row_len)])
            assert nb == len({s[0] for s in spans}) and len(spans) <= 3 * nb and len(spans) < rows
            assert sum(s[2] * s[3] for s in spans) == rows * row_len
        spans, nb, fetch = r.readv_strided_plan([(0, rows // world * pitch, 1, 0, 0, 0)])  # dim 0: one plain range, whole blocks direct
        assert len(spans) == nb and sum(1 for s in spans if s[5]) >= nb - 1


@pytest.mark.parametrize("rng_,what", [
    ((0, -1, 1, 0, 0), "negative length"),
    ((0, 10, -1, 10, 10), "negative row count"),
    ((0, 10, 2, -10, 10), "negative pitch"),
    ((0, 10, 1, 0, -1), "negative pitch"),
    ((0, 10, 2, 9, 10), "pitch shorter"),
    ((0, 10, 2, 10, 9), "pitch shorter"),
    ((0, 10, 1 << 62, 1 << 20, 10), "overflows"),
    ((0, 10, 3, 10, 1 << 62), "overflows"),
    ((0, 10, 100, 2 * BS, 10), "outside the file"),
    ((-1, 10, 1, 0, 0), "outside the file"),
    ((40 * BS - 1000, 2, 1, 0, 2), "outside the file"),
])
def test_malformed_strided_ranges_are_errors(files, rng_, what):
    fs, _ = files
    off, L, R, P, dp = rng_
    with fs.open("/sp/a") as r:
        with pytest.raises(F.FsError, match=r"range 0\b.*" + what) as e:
            r.readv_strided_plan([(off, L, R, P, 0, dp)])
        assert e.value.kind == 10000
        assert r.readv_strided_plan([(0, 10, 2, 20, 0, 10)])[1] == 1  # the reader is still usable


def test_overlapping_and_interleaved_ranges_are_errors(files):
    fs, _ = files
    with fs.open("/sp/a") as r:
        for rs in ([(0, 10, 5, 100, 0, 10), (50, 10, 5, 100, 0, 10)],   # interleaved rows: the extents overlap
                   [(0, 10, 5, 100, 0, 10), (405, 20, 1, 0, 0, 20)],    # a plain range over the last row
                   [(1000, 10, 1, 0, 0, 10), (0, 1, 11, 100, 0, 1)]):   # out of order
            with pytest.raises(F.FsError, match="overlap"):
                r.readv_strided_plan(rs)
        assert r.readv_strided_plan([(0, 10, 5, 100, 0, 10), (410, 10, 5, 100, 0, 10)])[1] == 1


def test_negative_count_and_missing_table_are_errors(files):
    fs, _ = files
    L = _lib.lib()
    with fs.open("/sp/a") as r:
        n = ctypes.c_int32()
        arr = (_lib.CvStridedRange * 1)()
        assert L.cv_readv_strided_plan(r._h, arr, -1, None, None, None, None, None, None, 0, None, None, None) == -10000
        assert b"negative range count" in L.cv_last_error()
        assert L.cv_readv_strided_plan(r._h, None, 2, None, None, None, None, None, None, 0, None, None, None) == -10000
        assert L.cv_readv_strided_plan(r._h, None, 0, None, None, None, None, None, None, 0, ctypes.byref(n), None, None) == 0 and n.value == 0
        nb = ctypes.c_int64()
        assert L.cv_readv_strided_device(r._h, None, 1, None, ctypes.byref(nb)) == -10000


# ---- safetensors.load_file(slices=...): validation and range construction (safetensors.plan_ranges)

def _entries():
    import torch
    ents = {"w": (torch.bfloat16, (6, 8), 0, 96), "b": (torch.float32, (8,), 96, 128), "t": (torch.int8, (2, 3, 4), 128, 152),
            "s": (torch.float64, (), 152, 160), "z": (torch.float16, (0, 4), 160, 160)}
    return 1000, ents


def test_slice_ranges_are_one_strided_range_per_tensor():
    start, ents = _entries()
    names = list(ents)
    got = {n: (shape, rng) for n, _, shape, rng in ST.plan_ranges(start, ents, names, {"w": (1, 2, 6), "t": (-1, 1, 3), "b": (0, 4, 8)})}
    assert got["w"] == ((6, 4), (1000 + 2 * 2, 4 * 2, 6, 8 * 2, 4 * 2))        # dim 1 of [6, 8] bf16: 6 rows of 8 bytes, 16 apart
    assert got["t"] == ((2, 3, 2), (1000 + 128 + 1, 2, 6, 4, 2))               # the last dim of [2, 3, 4] int8
    assert got["b"] == ((4,), (1000 + 96 + 16, 16, 1, 32, 16))                  # dim 0: one plain row
    assert got["s"] == ((), (1000 + 152, 8, 1, 0, 0)) and got["z"] == ((0, 4), None)
    got = {n: (shape, rng) for n, _, shape, rng in ST.plan_ranges(start, ents, names, {"w": (0, 3, 3), "z": (1, 0, 2)})}
    assert got["w"] == ((0, 8), None) and got["z"] == ((0, 2), None)           # empty slices read nothing
    got = {n: rng for n, _, _, rng in ST.plan_ranges(start, ents, ["w"], {"w": (0, 2, 5)})}
    assert got == {"w": (1000 + 2 * 16, 3 * 16, 1, 6 * 16, 3 * 16)}


@pytest.mark.parametrize("slices,err,what", [
    ({"nope": (0, 0, 1)}, KeyError, "nope"),
    ({"b": (0, 0, 1)}, ValueError, "not among the selected"),
    ({"s": (0, 0, 1)}, ValueError, "0-d"),
    ({"w": (2, 0, 1)}, ValueError, "out of range"),
    ({"w": (-3, 0, 1)}, ValueError, "out of range"),
    ({"w": (0, 4, 3)}, ValueError, "not a slice"),
    ({"w": (0, -1, 3)}, ValueError, "not a slice"),
    ({"w": (1, 0, 9)}, ValueError, "not a slice"),
    ({"w": (1, 0.0, 2)}, ValueError, "integers"),
    ({"w": (True, 0, 2)}, ValueError, "integers"),
    ({"w": (1, 2)}, ValueError, "integers"),
])
def test_malformed_slices_are_rejected(slices, err, what):
    start, ents = _entries()
    with pytest.raises(err, match=what):
        ST.plan_ranges(start, ents, ["w", "s"], slices)


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
        self.calls.append(ranges)
        return sum(r[1] * r[2] for r in ranges)

    def verify(self):
        return 0, 0, 0

    def complete(self):
        pass


def test_load_file_validates_before_reading_and_issues_one_call(monkeypatch):
    import torch
    from test_readv_plan import write_safetensors
    blob = write_safetensors([("w", "BF16", (6, 8), bytes(96)), ("b", "F32", (8,), bytes(32))])
    rd = _FakeReader(blob)
    fake_fs = type("FS", (), {"open": lambda self, p: rd})()
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: type("S", (), {"cuda_stream": 0})())
    allocs = []
    real_empty = torch.empty
    monkeypatch.setattr(torch, "empty", lambda *a, **k: allocs.append(a) or real_empty(*a, **{**k, "device": "cpu"}))
    for bad in ({"w": (5, 0, 1)}, {"nope": (0, 0, 1)}):
        with pytest.raises((ValueError, KeyError)):
            ST.load_file(fake_fs, "/x", device="cpu", slices=bad)
    assert not allocs and not rd.calls  # nothing allocated, nothing read
    out = ST.load_file(fake_fs, "/x", device="cpu", slices={"w": (1, 4, 8)})
    assert tuple(out["w"].shape) == (6, 4) and tuple(out["b"].shape) == (8,) and len(rd.calls) == 1
    (w, b), start = rd.calls[0], len(blob) - 128
    assert w[:4] == (start + 8, 8, 6, 16) and w[5] == 8 and b[:4] == (start + 96, 32, 1, 0)
    assert ST.read_header(fake_fs, "/x") == {"w": (torch.bfloat16, (6, 8)), "b": (torch.float32, (8,))}
