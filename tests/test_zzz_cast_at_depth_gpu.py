"""K5 at the grid depth real loads reach.  cvk_gather_cast and cvk_gather_cast_scaled are launched directly with one table shaped like
the ones the reader's scatter emits at 4 MiB blocks: long one-row spans (up to 1 Mi elements), spans of thousands of rows of 256..2048
elements, spans of up to a million rows of 1..7 elements (where the head chunk dominates), a run of thousands of one-row segments of
a few elements, and empty segments (no elements or no rows) at the start, in the middle and at the end.  launch_cast caps the grid
at SMs x 8 CTAs of 256 threads (270,336 threads on an H100's 132 SMs), so every thread walks many chunks and each grid stride skips
many segments through the forward segment search.

The whole destination (rows and the guard bytes between them) is compared with torch on the CPU, segment by segment: the plain
instance over all six F32/F16/BF16 pairs, the scaled one over E4M3/E5M2 into all three destination types with float32 block scales.
Each call is exactly one launch.

Depth, from the seeded table (chunks per thread = the table's chunks / the launched threads):
  H100:        4,135 segments, 70.8 Mi elements, 35.5 M chunks over 270,336 threads: 131 chunks per thread
  stand-ins:   the host-side shim (tests/simt_emu) reports 132 SMs too, so the cap is the same; a full-depth table is too slow on host
               cores, so the depth comes from the shape: 65,551 segments, most of them one-row segments of 2..9 elements (two chunks
               each), 270 K elements, 143 K chunks over 34,048 threads: 4.2 chunks per thread, each grid stride skipping about 17,000
               segments."""
import numpy as np
import pytest

from curvine_b200 import _lib
from test_zzz_readv_cast_gpu import GUARD, MOCK
from test_zzz_readv_scaled_gpu import _code, _scales

pytestmark = pytest.mark.gpu

FLOATS = ["float32", "float16", "bfloat16"]
PAIRS = [(a, b) for a in FLOATS for b in FLOATS if a != b]
F8 = ["float8_e4m3fn", "float8_e5m2"]
SMS_ON_STAND_INS = 132
# scale geometries (view cols, block_rows, block_cols): 128 x 128 tiles of a 5000-wide weight, one scale per row, small tiles
GEOMETRIES = [(5000, 128, 128), (777, 1, 777), (96, 16, 8)]


def _torch():
    import torch
    return torch


def _int(dt):
    torch = _torch()
    return {1: torch.uint8, 2: torch.int16, 4: torch.int32}[dt.itemsize]


class Table:
    """the segments in ELEMENTS: src_e, dst_e, elems, rows, src pitch, dst pitch, and the scale geometry index; `run` is the slice of
    the one-row run (checked vectorised)"""

    def __init__(self, full, seed=5):
        rng = np.random.default_rng(seed)
        self.cols = []
        self.src_n = self.dst_n = 64
        empties = lambda: [(0, 3), (5, 0), (0, 0)]  # noqa: E731  (elems, rows)
        parts = []
        if full:
            parts += [("one", int(rng.integers(256 << 10, (1 << 20) + 1)), 1) for _ in range(8)]
            parts += [("multi", int(rng.integers(256, 2049)), int(rng.integers(1000, 4001))) for _ in range(6)]
            parts += [("multi", int(rng.choice([1, 2, 2, 3, 3, 4, 5, 6, 7])), int(rng.integers(800 << 10, 1200 << 10))) for _ in range(16)]
            run = (4096, [1, 2, 3, 4, 5, 6, 7])
        else:
            parts += [("one", int(rng.integers(3000, 5000)), 1) for _ in range(2)]
            parts += [("multi", int(rng.integers(256, 300)), 40) for _ in range(2)]
            parts += [("multi", int(rng.integers(2, 8)), 2000) for _ in range(2)]
            run = (1 << 16, [2, 2, 2, 2, 2, 3, 5, 9])
        rng.shuffle(parts)
        half = len(parts) // 2
        for e, r in empties():
            self._add(rng, e, r)
        for kind, e, r in parts[:half]:
            self._add(rng, e, r)
        self._run(rng, *run)
        for e, r in empties():
            self._add(rng, e, r)
        for kind, e, r in parts[half:]:
            self._add(rng, e, r)
        for e, r in empties():
            self._add(rng, e, r)
        self.t = np.array(self.cols, dtype=np.int64)
        self.src_n += 64
        self.dst_n += 64

    def _add(self, rng, elems, rows):
        src = self.src_n + int(rng.integers(0, 8))
        dst = self.dst_n + int(rng.integers(0, 8))  # every phase of the destination against 16 bytes: every head length
        sp = elems + int(rng.integers(0, 4)) if rows > 1 else 0
        dp = elems + int(rng.integers(1, 5)) if rows > 1 else 0  # at least one guard element between two rows
        self.cols.append((src, dst, elems, rows, sp, dp, int(rng.integers(0, len(GEOMETRIES)))))
        if elems and rows:
            self.src_n = src + (rows - 1) * sp + elems + int(rng.integers(1, 9))
            self.dst_n = dst + (rows - 1) * dp + elems + int(rng.integers(1, 9))

    def _run(self, rng, m, lengths):
        e = rng.choice(np.array(lengths, dtype=np.int64), size=m)
        src = self.src_n + np.concatenate([[0], np.cumsum(e + rng.integers(0, 4, m))[:-1]])
        dst = self.dst_n + np.concatenate([[0], np.cumsum(e + rng.integers(1, 5, m))[:-1]])
        g = int(rng.integers(0, len(GEOMETRIES)))
        a = len(self.cols)
        self.cols += [(int(s), int(d), int(k), 1, 0, 0, g) for s, d, k in zip(src, dst, e)]
        self.run = slice(a, len(self.cols))
        self.src_n, self.dst_n = int(src[-1] + e[-1]) + 8, int(dst[-1] + e[-1]) + 8

    def chunks(self):
        e, r = self.t[:, 2], self.t[:, 3]
        return r * np.where(e > 0, (e + 14) // 8, 0)

    def elems(self):
        return int((self.t[:, 2] * self.t[:, 3]).sum())


def _threads(table):
    """the threads launch_cast starts for this table"""
    torch = _torch()
    sms = SMS_ON_STAND_INS if MOCK else torch.cuda.get_device_properties(0).multi_processor_count
    return min(table.elems() // 2048 + 1, sms * 8) * 256


def _packed(lo, hi):
    return (np.asarray(lo, dtype=np.int64) & 0xFFFFFFFF) | (np.asarray(hi, dtype=np.int64) << 32)


def _tables(table, ss, ds, sdt, ddt, scale_ptrs, dev):
    """-> (CvCastSeg table, CvScaleSeg table or None) on `dev`, built from the element table without a Python loop per segment"""
    torch = _torch()
    t = table.t
    ch = table.chunks()
    first = np.concatenate([[0], np.cumsum(ch)[:-1]])
    cast = np.stack([t[:, 0] * ss, t[:, 1] * ds, t[:, 2], t[:, 3], t[:, 4] * ss, t[:, 5] * ds, first,
                     _packed(np.full(len(t), sdt), np.full(len(t), ddt))], axis=1)
    d_cast = torch.from_numpy(cast.astype(np.int64)).view(torch.uint8).reshape(-1).to(dev)
    if scale_ptrs is None:
        return d_cast, None
    geo = np.array(GEOMETRIES, dtype=np.int64)[t[:, 6]]
    cols, br, bc = geo[:, 0], geo[:, 1], geo[:, 2]
    ptr = np.array(scale_ptrs, dtype=np.uint64).view(np.int64)[t[:, 6]]
    # the view: the source seen as one weight per geometry; a segment row k starts at view element src_e + k * src pitch
    sc = np.stack([ptr, br, bc, -(-cols // bc), cols, t[:, 0], t[:, 4], _packed(np.full(len(t), _lib.DTYPE_F32), np.zeros(len(t)))], axis=1)
    return d_cast, torch.from_numpy(sc.astype(np.int64)).view(torch.uint8).reshape(-1).to(dev)


def _finite_source(n, dt, seed):
    """n random elements of dt with every NaN pattern made finite (flip the exponent's top bit), so whole buffers compare bit for bit"""
    torch = _torch()
    raw = torch.from_numpy(np.random.default_rng(seed).integers(0, 256, size=n * dt.itemsize, dtype=np.uint8))
    nan = torch.isnan(raw.view(dt).float())
    iv = raw.view(_int(dt))
    iv[nan] ^= {1: 0x40, 2: 0x4000, 4: 0x40000000}[dt.itemsize]
    assert not bool(torch.isnan(raw.view(dt).float()).any())
    return raw


def _scale_tensors(table, seed):
    torch = _torch()
    rng = np.random.default_rng(seed)
    out = []
    for cols, br, bc in GEOMETRIES:
        n = (table.src_n // cols // br + 1) * -(-cols // bc)
        out.append(_scales(rng, n, torch.float32).float())  # random magnitudes of both signs, zeros, products that overflow or are denormal
    return out


def _expected(table, src, sdt, ddt, scales):
    """the destination on the CPU: guard bytes, and each segment's rows converted by torch"""
    torch = _torch()
    want = torch.full((table.dst_n * ddt.itemsize,), GUARD, dtype=torch.uint8)
    wt, st = want.view(_int(ddt)), src.view(sdt)

    def convert(x, v, g):
        if scales is None:
            return x.to(ddt)
        cols, br, bc = GEOMETRIES[g]
        idx = (v // cols // br) * -(-cols // bc) + (v % cols) // bc
        return (x.float() * scales[g][idx]).to(ddt)

    run = table.t[table.run]
    for i, (s, d, e, r, sp, dp, g) in enumerate(table.t.tolist()):
        if table.run.start <= i < table.run.stop or not (e and r):
            continue
        x = st.as_strided((r, e), (sp, 1), s)
        v = s + torch.arange(r, dtype=torch.int64)[:, None] * sp + torch.arange(e, dtype=torch.int64)[None, :]
        wt.as_strided((r, e), (dp, 1), d).copy_(convert(x, v, g).view(_int(ddt)))
    e = run[:, 2]
    local = np.arange(int(e.sum())) - np.repeat(np.cumsum(e) - e, e)
    si, di = torch.from_numpy(np.repeat(run[:, 0], e) + local), torch.from_numpy(np.repeat(run[:, 1], e) + local)
    wt[di] = convert(st[si], si, int(run[0, 6])).view(_int(ddt))
    return want


def _check(table, got, want, ddt, what):
    """got == want bit for bit, except that a NaN only has to stay a NaN (an FP8 infinity times a zero scale); on a mismatch, the
    segment whose destination holds the first bad element"""
    torch = _torch()
    if bool(torch.equal(got, want)):
        return
    g, w = got.view(ddt), want.view(ddt)
    nan = torch.isnan(w.float())
    bad = np.flatnonzero(((g.view(_int(ddt)) != w.view(_int(ddt))) & ~nan).numpy()) * ddt.itemsize
    assert bool(torch.isnan(g.float()[nan]).all()), what
    if not bad.size:
        return
    ds = ddt.itemsize
    seg = int(np.searchsorted(table.t[:, 1] * ds, bad[0], side="right")) - 1
    assert False, (what, "%d bytes differ, the first at byte %d, in or after segment %d %s" % (bad.size, bad[0], seg, table.t[seg].tolist()))


@pytest.fixture(scope="module")
def table():
    t = Table(full=not MOCK)
    print("K5 depth table: %d segments, %d elements, %d chunks over %d threads: %.1f chunks per thread"
          % (len(t.t), t.elems(), int(t.chunks().sum()), _threads(t), t.chunks().sum() / _threads(t)))
    return t


def test_the_table_reaches_the_depth_it_is_there_for(table):
    """the docstring's numbers: the table keeps them if its generator changes"""
    depth = table.chunks().sum() / _threads(table)
    assert depth >= (4 if MOCK else 120), depth
    assert len(table.t) >= (1 << 16 if MOCK else 4096)
    assert MOCK or table.elems() >= 64 << 20
    e, r = table.t[:, 2], table.t[:, 3]
    empty = np.flatnonzero((e == 0) | (r == 0))
    assert empty[0] == 0 and empty[-1] == len(e) - 1 and ((empty > 3) & (empty < len(e) - 4)).any()


def _launch(table, src_dt, dst_dt, scaled, seed):
    torch = _torch()
    from curvine_b200 import kernels as K
    dev = torch.device("cpu") if MOCK else torch.device("cuda", 0)
    src = _finite_source(table.src_n, src_dt, seed)
    scales = _scale_tensors(table, seed + 1) if scaled else None
    d_scales = [s.to(dev) for s in scales] if scaled else None
    d_cast, d_sc = _tables(table, src_dt.itemsize, dst_dt.itemsize, _code(src_dt), _code(dst_dt),
                           [s.data_ptr() for s in d_scales] if scaled else None, dev)
    d_src = src.to(dev)
    dst = torch.full((table.dst_n * dst_dt.itemsize,), GUARD, dtype=torch.uint8, device=dev)
    before = K.launch_count()
    if scaled:
        K.gather_cast_scaled(d_src, d_cast, d_sc, len(table.t), table.elems(), dst)
    else:
        K.gather_cast(d_src, d_cast, len(table.t), table.elems(), dst)
    assert K.launch_count() == before + 1
    got = dst.cpu()
    del d_src, dst, d_scales
    return got, _expected(table, src, src_dt, dst_dt, scales)


@pytest.mark.parametrize("src_name,dst_name", PAIRS)
def test_plain_instance_at_full_grid_depth(cuda, table, src_name, dst_name):
    torch = _torch()
    got, want = _launch(table, getattr(torch, src_name), getattr(torch, dst_name), False, 7 + PAIRS.index((src_name, dst_name)))
    _check(table, got, want, getattr(torch, dst_name), (src_name, dst_name))


@pytest.mark.parametrize("dst_name", FLOATS)
@pytest.mark.parametrize("src_name", F8)
def test_scaled_instance_at_full_grid_depth(cuda, table, src_name, dst_name):
    torch = _torch()
    got, want = _launch(table, getattr(torch, src_name), getattr(torch, dst_name), True, 31 + F8.index(src_name) * 3 + FLOATS.index(dst_name))
    _check(table, got, want, getattr(torch, dst_name), (src_name, dst_name))
