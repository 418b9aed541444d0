"""The newer kernels checked in isolation (the product paths that use them -- small-file reads, FUSE page scatter, the 262,144-page
kbench case -- are covered by the reader suites too).  The file sorts after the established suites on purpose: whatever happens here,
everything else has already run.

  * crc_small_kernel / gather_small_kernel: the single-launch small-input kernels, against the oracle and against the launch train
  * the multi-CTA prefix scan (more than 16 Ki pieces)"""
import os
import zlib

import numpy as np
import pytest

from oracle import clib
from test_kernels_gpu import _rand, _to_dev

pytestmark = pytest.mark.gpu


SMALL_LENS = [0, 1, 2, 3, 4, 5, 7, 8, 15, 16, 17, 31, 33, 1023, 1024, 1025, 4095, 4096, 4097, 16383, 16384, 16385, 65536 + 7, 131072, 262144,
              262144 + 5, 1024 * 1008 - 1, 1024 * 1008]


@pytest.mark.parametrize("poly", [0, 1])
@pytest.mark.parametrize("small_path", [1, 0])
def test_crc_small_inputs_single_launch_kernel_vs_launch_train(cuda, poly, small_path):
    """Inputs of at most ~1 MiB take the single-launch kernel (crc_small_kernel: slicing-by-4 chunk CRCs, init folded into the first
    four bytes, pairwise combine with squared multipliers); cvk_tune(5, 0) sends the same inputs through the general launch train.
    Both must equal the oracle at every length and base alignment, one block per launch and several blocks per launch."""
    from curvine_b200 import _lib, kernels as K
    data = _rand((1 << 20) + 4096, 4321 + poly)
    d = _to_dev(data, cuda)
    _lib.check(_lib.lib().cvk_tune(5, small_path))
    try:
        before = K.launch_count()
        for n in SMALL_LENS:
            for mis in (0, 1, 3, 6):
                got = K.u32(K.crc_blocks(d, [mis], [n], poly))
                assert int(got[0]) == clib.crc(poly, data[mis:mis + n]), (n, mis)
        if small_path:
            assert K.launch_count() - before == 4 * len([n for n in SMALL_LENS])  # exactly one launch per call
        # several small blocks in one launch (a read_many batch / a verify batch of small files)
        offs, lens, pos = [], [], 5
        for n in [0, 1, 3, 4, 100, 4096, 65536 + 1, 200000, 262144, 300001]:
            offs.append(pos)
            lens.append(n)
            pos += n + 11
        got = K.u32(K.crc_blocks(d, offs, lens, poly))
        assert got.tolist() == [clib.crc(poly, data[o:o + n]) for o, n in zip(offs, lens)]
    finally:
        _lib.check(_lib.lib().cvk_tune(5, 1))


@pytest.mark.parametrize("small_path", [1, 0])
def test_gather_small_inputs_single_launch_kernel(cuda, small_path):
    """A FUSE reply's worth of pages (<= 1 MiB) scatters in one launch (gather_small_kernel): aligned vectors, same-phase words and
    byte-wise segments all equal the byte-exact model."""
    import torch
    from curvine_b200 import _lib, kernels as K
    src = _rand(1 << 20, 77)
    d_src = _to_dev(src, cuda)
    _lib.check(_lib.lib().cvk_tune(5, small_path))
    try:
        for shape in ("aligned", "same_phase", "bytes", "ragged"):
            segs, pos = [], 0
            for i in range(64):
                n = 4096 if shape != "ragged" else [0, 1, 15, 16, 17, 4095, 4096, 333][i % 8]
                so = {"aligned": i * 4096, "same_phase": i * 4096 + 6, "bytes": i * 4096 + 5, "ragged": i * 4099 + (i % 7)}[shape]
                do = {"aligned": (63 - i) * 4096, "same_phase": (63 - i) * 4100 + 2, "bytes": (63 - i) * 4100 + 2, "ragged": pos}[shape]
                segs.append((so, do, n))
                pos += n + (i % 3)
            size = max(do + n for _, do, n in segs) + 32
            want = np.full(size, 0xC3, dtype=np.uint8)
            for so, do, n in segs:
                want[do:do + n] = src[so:so + n]
            dst = torch.full((size,), 0xC3, dtype=torch.uint8, device=cuda)
            before = K.launch_count()
            K.gather_pages(d_src, K.segs_to_device(segs, cuda), len(segs), sum(x[2] for x in segs), dst)
            assert dst.cpu().numpy().tobytes() == want.tobytes(), shape
            if small_path:
                assert K.launch_count() - before == 1
    finally:
        _lib.check(_lib.lib().cvk_tune(5, 1))


@pytest.mark.parametrize("n_segs", [16384, 16385, 20480, 40003])
def test_more_than_16k_pieces_take_the_multi_cta_scan(cuda, n_segs):
    """tile_sums_kernel + scan_tiles_kernel: same check as test_kernels_gpu.test_many_small_pieces_multi_tile_scan, above the switch-over."""

    import torch
    from curvine_b200 import kernels as K
    rng = np.random.default_rng(n_segs)
    src = _rand(1 << 20, 12)
    lens = rng.choice([0, 1, 7, 16, 33, 100, 257, 4096], size=n_segs)
    sos = rng.integers(0, len(src) - 4096, size=n_segs)
    segs, pos = [], 0
    for so, n in zip(sos, lens):
        segs.append((int(so), pos, int(n)))
        pos += int(n) + int(rng.integers(0, 3))
    want = np.zeros(pos + 16, dtype=np.uint8)
    for so, do, n in segs:
        want[do:do + n] = src[so:so + n]
    d_src = _to_dev(src, cuda)
    dst = torch.zeros(pos + 16, dtype=torch.uint8, device=cuda)
    K.gather_pages(d_src, K.segs_to_device(segs, cuda), len(segs), int(lens.sum()), dst)
    assert dst.cpu().numpy().tobytes() == want.tobytes()
    got = K.u32(K.crc_blocks(d_src, [int(x) for x in sos], [int(x) for x in lens], 1))
    assert got.tolist() == [clib.crc(1, src[o:o + n]) for o, n in zip(sos, lens)]


VARIANTS = [("seg_4k", [(4, 12)]), ("seg_64k", [(4, 16)])]


@pytest.mark.parametrize("name,tunes", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_every_walker_variant_is_bit_identical(cuda, name, tunes):
    """cvk_tune(4, s) forces a segment size the launchers otherwise derive from the input size: with it, K2 (unpack: every source
    phase, since 22-byte prefixes rotate it), K4 (pack) and K3 (gather, every source/destination phase pair) must produce the
    bytes and CRCs of the oracle."""
    import torch
    from curvine_b200 import _lib, kernels as K
    from oracle import wire as W
    from test_kernels_gpu import _build_wire
    L = _lib.lib()
    try:
        for what, value in tunes:
            _lib.check(L.cvk_tune(what, value))
        _lib.check(L.cvk_tune(5, 0))  # the launch train, not the small-input kernels
        for poly in (0, 1):
            blocks = [_rand(n, 300 + i) for i, n in enumerate([70000, 4096, 1, 131072 + 9, 33, 250000])]
            chunk = 8192 + 16  # 22-byte prefixes + this chunk walk the payloads through source phases 6, 12, 2, 8, ...
            wire, descs, _, total = _build_wire(blocks, chunk, [900 + i for i in range(len(blocks))], poly)
            want = np.concatenate(blocks)
            want_crc = [clib.crc(poly, b) for b in blocks]
            d_desc = K.frame_descs_to_device(descs, cuda)
            for mis in (0, 5):
                dst = torch.full((total + mis + 48,), 0x5A, dtype=torch.uint8, device=cuda)
                crc, err = K.unpack_frames(_to_dev(wire, cuda), d_desc, len(descs), len(blocks), dst[mis:], poly, total)
                out = dst.cpu().numpy()
                assert out[mis:mis + total].tobytes() == want.tobytes() and (out[:mis] == 0x5A).all() and (out[mis + total:] == 0x5A).all(), (name, poly, mis)
                assert K.u32(crc).tolist() == want_crc and (K.u32(err) == 0).all()
            d_wire = torch.zeros(len(wire), dtype=torch.uint8, device=cuda)
            crc = K.pack_frames(_to_dev(want, cuda), d_desc, len(descs), len(blocks), d_wire, poly, total)
            assert d_wire.cpu().numpy().tobytes() == wire.tobytes() and K.u32(crc).tolist() == want_crc
            msgs, used = W.decode_stream(d_wire.cpu().numpy().tobytes())
            assert used == len(wire) and b"".join(m.data for m in msgs) == want.tobytes()
        src = _rand(2 << 20, 55)
        segs, pos = [], 3
        for i in range(96):  # all 16 x 16 phase pairs show up: sources step by 4099 + i, destinations by n + i % 5
            n = [40000, 4096, 17, 16, 15, 1, 0, 70001][i % 8]
            segs.append((i * 4099 + i, pos, n))
            pos += n + i % 5
        wantb = np.full(pos + 32, 0xA5, dtype=np.uint8)
        for so, do, n in segs:
            wantb[do:do + n] = src[so:so + n]
        dst = torch.full((pos + 32,), 0xA5, dtype=torch.uint8, device=cuda)
        K.gather_pages(_to_dev(src, cuda), K.segs_to_device(segs, cuda), len(segs), sum(s[2] for s in segs), dst)
        assert dst.cpu().numpy().tobytes() == wantb.tobytes(), name
    finally:
        for what, value in ((4, 0), (5, 1)):
            L.cvk_tune(what, value)


def test_gather_and_frames_hypothesis_random_shapes(cuda):
    """Generated shapes for the DST walkers: K3 with random (source offset, length, gap) segments -- every source/destination phase,
    empty, sub-vector and multi-segment pieces, small-input kernel and launch train -- and K2/K4 with random block lengths and chunk
    sizes (the 22-byte prefixes rotate the source phase frame by frame).  Bytes, untouched gaps and CRCs against numpy / the oracle."""
    import torch
    from hypothesis import given, settings, strategies as st
    from curvine_b200 import _lib, kernels as K
    from test_kernels_gpu import _build_wire
    src = _rand(1 << 20, 91)
    d_src = _to_dev(src, cuda)
    L = _lib.lib()
    scale = int(os.environ.get("CV_TEST_HYPOTHESIS_SCALE", "1"))  # a long hunt on the host-side shim: CV_TEST_HYPOTHESIS_SCALE=50

    @settings(max_examples=30 * scale, deadline=None)
    @given(st.lists(st.tuples(st.integers(0, (1 << 20) - 70000), st.sampled_from([0, 1, 2, 15, 16, 17, 31, 100, 511, 512, 513, 4096, 5000, 20000, 66000]),
                              st.integers(0, 19)), min_size=1, max_size=40), st.integers(0, 15), st.booleans())
    def gather(items, first, small):
        segs, pos = [], first
        for so, n, gap in items:
            segs.append((so, pos, n))
            pos += n + gap
        want = np.full(pos + 16, 0x3C, dtype=np.uint8)
        for so, do, n in segs:
            want[do:do + n] = src[so:so + n]
        dst = torch.full((pos + 16,), 0x3C, dtype=torch.uint8, device=cuda)
        _lib.check(L.cvk_tune(5, 1 if small else 0))
        K.gather_pages(d_src, K.segs_to_device(segs, cuda), len(segs), sum(s[2] for s in segs), dst)
        assert dst.cpu().numpy().tobytes() == want.tobytes()

    @settings(max_examples=20 * scale, deadline=None)
    @given(st.lists(st.integers(1, 90000), min_size=1, max_size=6), st.sampled_from([1, 7, 16, 100, 4096, 4100, 65536]), st.integers(0, 1), st.integers(0, 15))
    def frames(blens, chunk, poly, mis):
        blens = [min(n, chunk * 40) for n in blens]  # at most 40 frames per block keeps an example small
        blocks = [_rand(n, 700 + i) for i, n in enumerate(blens)]
        wire, descs, _, total = _build_wire(blocks, chunk, [31 + i for i in range(len(blocks))], poly)
        want = np.concatenate(blocks)
        d_desc = K.frame_descs_to_device(descs, cuda)
        dst = torch.full((total + mis + 32,), 0x99, dtype=torch.uint8, device=cuda)
        crc, err = K.unpack_frames(_to_dev(wire, cuda), d_desc, len(descs), len(blocks), dst[mis:], poly, total)
        out = dst.cpu().numpy()
        assert out[mis:mis + total].tobytes() == want.tobytes() and (out[:mis] == 0x99).all() and (out[mis + total:] == 0x99).all()
        assert K.u32(crc).tolist() == [clib.crc(poly, b) for b in blocks] and (K.u32(err) == 0).all()
        d_wire = torch.zeros(len(wire), dtype=torch.uint8, device=cuda)
        crc = K.pack_frames(_to_dev(want, cuda), d_desc, len(descs), len(blocks), d_wire, poly, total)
        assert d_wire.cpu().numpy().tobytes() == wire.tobytes() and K.u32(crc).tolist() == [clib.crc(poly, b) for b in blocks]

    try:
        gather()
        frames()
    finally:
        L.cvk_tune(5, 1)
