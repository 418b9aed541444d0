"""Vectored reads without a GPU: the plan cv_readv_device executes (cv_readv_plan) against a Python restatement of the block
classification, rejection of malformed range sets, and the safetensors header parser of curvine_b200.safetensors."""
import ctypes
import json
import os
import shutil
import struct
import tempfile

import numpy as np
import pytest

from curvine_b200 import _lib, fs as F
from curvine_b200 import safetensors as ST


def model_plan(ranges, block_lens):
    """-> (spans, n_blocks, fetch_bytes) as Reader.readv_plan returns them.  A block is direct when one range covers all of it."""
    starts = np.concatenate([[0], np.cumsum(block_lens)]).tolist()
    spans = []
    for i in sorted((i for i, r in enumerate(ranges) if r[1] > 0), key=lambda i: ranges[i][0]):
        p, end = ranges[i][0], ranges[i][0] + ranges[i][1]
        while p < end:
            b = next(b for b in range(len(block_lens)) if starts[b] <= p < starts[b + 1])
            take = min(end, starts[b + 1]) - p
            spans.append([b, p - starts[b], take, i])
            p += take
    blocks = {}
    for s in spans:
        blocks.setdefault(s[0], []).append(s)
    out = []
    for s in spans:
        mine = blocks[s[0]]
        out.append((s[0], s[1], s[2], s[3], len(mine) == 1 and s[1] == 0 and s[2] == block_lens[s[0]]))
    return out, len(blocks), sum(block_lens[b] for b in blocks)


def random_ranges(rng, n, max_ranges):
    """Non-overlapping ranges in random order, some empty, cut at random points of [0, n]."""
    cuts = sorted(set(int(x) for x in rng.integers(0, n + 1, size=2 * int(rng.integers(1, max_ranges + 1)))))
    pairs = [(a, b - a) for a, b in zip(cuts[::2], cuts[1::2])]
    pairs = [p for p in pairs if rng.random() < 0.8]
    pairs += [(int(rng.integers(0, n + 1)), 0)] * int(rng.integers(0, 2))
    rng.shuffle(pairs)
    return pairs


@pytest.fixture(scope="module")
def files():
    d = tempfile.mkdtemp(prefix="cvrp", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    w = F.MiniWorker(["[MEM]" + d + "/m"])
    bs = 64 << 10
    specs = {"/rp/short": ((10 * bs) - 999, 0), "/rp/holes": ((7 * bs) + 5, 3), "/rp/one": (bs // 2, 0)}
    mans = [w.create_file(p, 9500 + k, n, bs, mode=2 if he else 0, hole_every=he, threads=2) for k, (p, (n, he)) in enumerate(specs.items())]
    fs = F.CurvineFileSystem(F.client_conf())
    for m in mans:
        fs.load_namespace(m)
    yield fs, bs, {p: n for p, (n, _) in specs.items()}
    fs.close()
    w.stop()
    shutil.rmtree(d, ignore_errors=True)


def test_plan_matches_the_classification(files):
    fs, bs, sizes = files
    rng = np.random.default_rng(17)
    for path, n in sizes.items():
        lens = [min(bs, n - i) for i in range(0, n, bs)]
        fixed = [
            [(0, n)],                                     # the whole file: every block direct (the short last one too)
            [(bs, bs), (3 * bs, 2 * bs)],                 # exactly on block edges
            [(5, 1), (bs - 1, 1), (bs, 1), (n - 1, 1)],   # 1-byte ranges, either side of an edge
            [(10, 20), (40, 7), (100, bs - 200)],         # several ranges inside one block
            [(bs // 4, bs // 2)],                         # a range inside one block
            [(bs - 3, 6), (0, bs - 3), (bs + 3, 2 * bs)], # a block split between two ranges, out of order
            [(0, 0), (n, 0)],                             # empty ranges touch nothing
            [],
        ]
        sets = [[r for r in rs if r[0] + r[1] <= n] for rs in fixed] + [random_ranges(rng, n, 12) for _ in range(60)]
        with fs.open(path) as r:
            for rs in sets:
                got = r.readv_plan([(o, ln, 0) for o, ln in rs])
                assert got == model_plan(rs, lens), (path, rs)
                spans, nb, fetch = got
                assert sum(s[2] for s in spans) == sum(ln for _, ln in rs)
            assert r.pos() == 0


@pytest.mark.parametrize("ranges,what", [
    ([(0, 100), (50, 100)], "overlap"),
    ([(1000, 10), (0, 1001)], "overlap"),
    ([(0, 10), (5, 1)], "overlap"),
    ([(-1, 10)], "outside the file"),
    ([(0, (10 * (64 << 10)) - 998)], "outside the file"),
    ([((10 * (64 << 10)) - 999, 1)], "outside the file"),
    ([(1 << 62, 1 << 62)], "outside the file"),
    ([(0, -1)], "negative length"),
])
def test_malformed_ranges_are_errors(files, ranges, what):
    fs, _, _ = files
    with fs.open("/rp/short") as r:
        with pytest.raises(F.FsError, match=what) as e:
            r.readv_plan([(o, ln, 0) for o, ln in ranges])
        assert e.value.kind == 10000
        assert r.readv_plan([(0, 10, 0)])[1] == 1  # the reader is still usable


def test_negative_count_and_missing_table_are_errors(files):
    fs, _, _ = files
    L = _lib.lib()
    with fs.open("/rp/short") as r:
        arr = (_lib.CvRange * 1)()
        n = ctypes.c_int32()
        assert L.cv_readv_plan(r._h, arr, -1, None, None, None, None, None, 0, None, None, None) == -10000
        assert b"negative range count" in L.cv_last_error()
        assert L.cv_readv_plan(r._h, None, 3, None, None, None, None, None, 0, None, None, None) == -10000
        assert L.cv_readv_plan(r._h, None, 0, None, None, None, None, None, 0, ctypes.byref(n), None, None) == 0 and n.value == 0


# ---- safetensors header parser

def write_safetensors(tensors, metadata=None, pad_to=1):
    """tensors: list of (name, dtype name, shape, raw bytes) -> the file's bytes, data in list order."""
    header, data = {}, b""
    for name, dt, shape, raw in tensors:
        header[name] = {"dtype": dt, "shape": list(shape), "data_offsets": [len(data), len(data) + len(raw)]}
        data += raw
    if metadata is not None:
        header["__metadata__"] = metadata
    h = json.dumps(header).encode()
    h += b" " * (-(8 + len(h)) % pad_to)
    return struct.pack("<Q", len(h)) + h + data


def parse(blob):
    return ST.parse_header(lambda o, n: blob[o:o + n], len(blob))


def test_parser_accepts_well_formed_files():
    import torch
    t = [("w", "F32", (3, 4), bytes(48)), ("b", "BF16", (4,), bytes(8)), ("s", "I64", (), bytes(8)), ("e", "F16", (0, 5), b""),
         ("m", "BOOL", (2, 1), b"\x01\x00"), ("f8", "F8_E4M3", (3,), b"abc")]
    blob = write_safetensors(t, metadata={"format": "pt"}, pad_to=8)
    start, ents = parse(blob)
    assert start % 8 == 0 and start + 48 + 8 + 8 + 2 + 3 == len(blob)
    assert set(ents) == {"w", "b", "s", "e", "m", "f8"}
    assert ents["w"] == (torch.float32, (3, 4), 0, 48) and ents["s"][1] == () and ents["e"][2] == ents["e"][3]
    assert ents["f8"][0] == torch.float8_e4m3fn
    for name in ("U16", "U32", "U64"):
        if name in ST.dtypes():
            assert parse(write_safetensors([("u", name, (2,), bytes(2 * ST.dtypes()[name].itemsize))]))[1]["u"][1] == (2,)


def _hdr(obj, data=b"", raw=None):
    h = raw if raw is not None else json.dumps(obj).encode()
    return struct.pack("<Q", len(h)) + h + data


@pytest.mark.parametrize("blob,what", [
    (b"\x05\x00\x00", "too short"),
    (struct.pack("<Q", 50) + b"{}", "runs past the end"),
    (struct.pack("<Q", 1 << 62) + b"{}", "exceeds"),
    (_hdr(None, raw=b"{not json"), "not valid JSON"),
    (_hdr(None, raw=b"\xff\xfe{}"), "not valid JSON"),
    (_hdr(None, raw=b"[" * 100000 + b"]" * 100000), "not valid JSON|not a JSON object"),
    (_hdr([1, 2]), "not a JSON object"),
    (_hdr({"a": 5}), "not an object"),
    (_hdr({"a": {"dtype": "F33", "shape": [1], "data_offsets": [0, 4]}}, bytes(4)), "unknown dtype"),
    (_hdr({"a": {"dtype": "F32", "shape": [2], "data_offsets": [0, 4]}}, bytes(8)), "needs 8 bytes"),
    (_hdr({"a": {"dtype": "F32", "shape": [-1], "data_offsets": [0, 4]}}, bytes(4)), "shape"),
    (_hdr({"a": {"dtype": "F32", "shape": [True], "data_offsets": [0, 4]}}, bytes(4)), "shape"),
    (_hdr({"a": {"dtype": "F32", "shape": "1", "data_offsets": [0, 4]}}, bytes(4)), "shape"),
    (_hdr({"a": {"dtype": "F32", "shape": [1], "data_offsets": [0]}}, bytes(4)), "data_offsets"),
    (_hdr({"a": {"dtype": "F32", "shape": [1], "data_offsets": [0, 4.0]}}, bytes(4)), "data_offsets"),
    (_hdr({"a": {"dtype": "F32", "shape": [1], "data_offsets": [4, 8]}}, bytes(4)), "outside"),
    (_hdr({"a": {"dtype": "F32", "shape": [1], "data_offsets": [-4, 0]}}, bytes(4)), "outside"),
    (_hdr({"a": {"dtype": "F32", "shape": [0], "data_offsets": [4, 0]}}, bytes(4)), "outside"),
    (_hdr({"a": {"dtype": "F32", "shape": [2], "data_offsets": [0, 8]}, "b": {"dtype": "U8", "shape": [4], "data_offsets": [4, 8]}}, bytes(8)), "overlap"),
    (_hdr({"a": {"dtype": "F32", "shape": [1], "data_offsets": [0, 4]}, "b": {"dtype": "I32", "shape": [1], "data_offsets": [0, 4]}}, bytes(4)), "overlap"),
])
def test_parser_rejects_malformed_headers(blob, what):
    with pytest.raises(ST.SafetensorsError, match=what):
        parse(blob)
