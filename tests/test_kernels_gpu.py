"""Parity of the sm_90a kernels (through the C ABI) against the CPU oracle.  Bit-exact: integer/byte work."""
import zlib

import numpy as np
import pytest

from oracle import clib, wire as W
from oracle import crc as OC

pytestmark = pytest.mark.gpu

EDGE_LENS = [0, 1, 2, 3, 4, 5, 15, 16, 17, 31, 32, 33, 511, 512, 513, 1023, 4095, 4096, 4097,
             128 * 1024 - 1, 128 * 1024, 128 * 1024 + 1, (1 << 22) - 1, 1 << 22, (1 << 22) + 1]


def _rand(n, seed):
    return np.random.default_rng(seed).integers(0, 256, size=n, dtype=np.uint8)


def _to_dev(a, dev):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


@pytest.mark.parametrize("poly", [0, 1])
def test_crc_check_values(cuda, poly):
    from curvine_b200 import kernels as K
    d = _to_dev(np.frombuffer(b"123456789", dtype=np.uint8).copy(), cuda)
    got = K.u32(K.crc_blocks(d, [0], [9], poly))
    assert got[0] == (OC.CHECK_IEEE if poly == 0 else OC.CHECK_CASTAGNOLI)


@pytest.mark.parametrize("poly", [0, 1])
@pytest.mark.parametrize("misalign", [0, 1, 7, 13])
def test_crc_edge_lengths_and_alignment(cuda, poly, misalign):
    """Lengths {0,1,15,16,17,4095,4096,128Ki+-1,2^22+-1} at unaligned base pointers, one launch."""
    from curvine_b200 import kernels as K
    offs, lens, pos = [], [], misalign
    for n in EDGE_LENS:
        offs.append(pos)
        lens.append(n)
        pos += n + 3  # keep every block at a different alignment
    data = _rand(pos + 64, 1234 + misalign)
    got = K.u32(K.crc_blocks(_to_dev(data, cuda), offs, lens, poly))
    want = np.array([clib.crc(poly, data[o:o + n]) for o, n in zip(offs, lens)], dtype=np.uint32)
    assert (got == want).all(), [(n, hex(g), hex(w)) for n, g, w in zip(lens, got, want) if g != w]
    if poly == 0:  # the reference's own function: crc32fast::hash == zlib.crc32
        assert all(int(g) == zlib.crc32(data[o:o + n].tobytes()) for g, o, n in zip(got, offs, lens))


@pytest.mark.parametrize("poly", [0, 1])
def test_crc_many_uniform_blocks(cuda, poly):
    """C1-shaped: 64 MiB, 1 MiB blocks; and ragged last block."""
    from curvine_b200 import kernels as K
    total, bs = 64 * 1024 * 1024 - 12345, 1 << 20
    data = _rand(total, 99)
    n = (total + bs - 1) // bs
    offs = [i * bs for i in range(n)]
    lens = [min(bs, total - o) for o in offs]
    got = K.u32(K.crc_blocks(_to_dev(data, cuda), offs, lens, poly))
    assert (got == clib.crc_blocks(poly, data, bs)).all()


def test_crc_bench_style_sum(cuda):
    """curvine-bench figure: u64 sum of crc32 over 128 KiB buffers (curvine_bench.rs:37-48,222-231)."""
    from curvine_b200 import kernels as K
    total, bs = 16 * 1024 * 1024, 128 * 1024
    data = _rand(total, 5)
    offs = list(range(0, total, bs))
    got = K.u32(K.crc_blocks(_to_dev(data, cuda), offs, [bs] * len(offs), 0))
    assert int(got.astype(np.uint64).sum()) == clib.bench_checksum(data, bs)


def test_crc_linearity_property_large(cuda):
    """Size-independent property at a large size: CRC(A||B) == combine(CRC(A), CRC(B), |B|); CRC(A xor B) linear."""
    import torch
    from curvine_b200 import kernels as K
    n = 1 << 28
    g = torch.Generator(device=cuda).manual_seed(7)
    a = torch.randint(0, 256, (n,), dtype=torch.uint8, device=cuda, generator=g)
    cut = n // 3 + 5
    whole, pa, pb = K.u32(K.crc_blocks(a, [0, 0, cut], [n, cut, n - cut], 0))
    assert OC.crc_combine(int(pa), int(pb), n - cut, OC.POLY_IEEE) == int(whole)
    b = torch.randint(0, 256, (n,), dtype=torch.uint8, device=cuda, generator=g)
    z = torch.zeros(n, dtype=torch.uint8, device=cuda)
    ca, cb, cx, cz = (int(K.u32(K.crc_blocks(t, [0], [n], 1))[0]) for t in (a, b, a ^ b, z))
    assert ca ^ cb ^ cx == cz  # affine: crc(a)^crc(b)^crc(a^b) == crc(0...)


def test_verify_crcs(cuda):
    import torch
    from curvine_b200 import kernels as K
    crc = torch.arange(1000, dtype=torch.int32, device=cuda)
    exp = crc.clone()
    exp[[3, 500, 999]] += 1
    n_bad = torch.zeros(1, dtype=torch.int32, device=cuda)
    mask = torch.zeros(1000, dtype=torch.uint8, device=cuda)
    K.verify_crcs(crc, exp, n_bad, mask)
    assert int(n_bad.item()) == 3 and mask.cpu().numpy().nonzero()[0].tolist() == [3, 500, 999]


def _build_wire(blocks, chunk, req_ids, poly, bad=None):
    """Pipelined response streams of several blocks back to back, as the worker would send them."""
    from curvine_b200._lib import CvFrameDesc, CvStreamDesc
    wire, descs, streams, dst_off, fidx = bytearray(), [], [], 0, 0
    for b, (blk, rid) in enumerate(zip(blocks, req_ids)):
        streams.append(CvStreamDesc(len(wire), dst_off, len(blk), rid, chunk, 1, b, fidx, W.RPC_CODE_READ_BLOCK, 0x03))
        pos, seq = 0, 0
        while pos < len(blk):
            seq += 1
            n = min(chunk, len(blk) - pos)
            m = W.success(W.request(W.RPC_CODE_READ_BLOCK, W.REQ_RUNNING, rid, seq), b"", blk[pos:pos + n].tobytes())
            descs.append(CvFrameDesc(len(wire), dst_off + pos, n, 0, rid, seq, b, W.RPC_CODE_READ_BLOCK, 0x03))
            wire += W.encode(m)
            pos += n
            fidx += 1
        dst_off += len(blk)
    return np.frombuffer(bytes(wire), dtype=np.uint8).copy(), descs, streams, dst_off


@pytest.mark.parametrize("poly", [0, 1])
@pytest.mark.parametrize("chunk,blens", [(131072, [1 << 20, 1 << 20, (1 << 20) - 77]), (4096, [12345, 1, 4096, 8191]),
                                         (1 << 20, [4 << 20, (4 << 20) + 5])])
def test_unpack_frames_matches_oracle(cuda, poly, chunk, blens):
    """K2: payload bytes land at their file offsets, per-block CRC equals the oracle's, prefixes validate."""
    import torch
    from curvine_b200 import kernels as K
    blocks = [_rand(n, 10 + i) for i, n in enumerate(blens)]
    wire, descs, streams, total = _build_wire(blocks, chunk, [0x0102030405060708 + i for i in range(len(blocks))], poly)
    # oracle decode of the same wire image
    msgs, used = W.decode_stream(wire.tobytes())
    assert used == len(wire) and b"".join(m.data for m in msgs) == b"".join(b.tobytes() for b in blocks)
    d_wire = _to_dev(wire, cuda)
    for misalign in (0, 3):  # destination alignment
        dst = torch.zeros(total + 64, dtype=torch.uint8, device=cuda)
        d_desc = K.frame_descs_to_device(descs, cuda)
        crc, err = K.unpack_frames(d_wire, d_desc, len(descs), len(blocks), dst[misalign:], poly, total)
        assert (K.u32(err) == 0).all()
        assert dst[misalign:misalign + total].cpu().numpy().tobytes() == b"".join(b.tobytes() for b in blocks)
        assert K.u32(crc).tolist() == [clib.crc(poly, b) for b in blocks]
    # closed-form stream descriptors expand to the same table
    d_streams = K.stream_descs_to_device(streams, cuda)
    exp = K.expand_streams(d_streams, len(streams), len(descs), cuda)
    assert exp.cpu().numpy().tobytes() == K.frame_descs_to_device(descs, cuda).cpu().numpy().tobytes()


@pytest.mark.parametrize("clip", [1, 15, 16, 4095, 4096])
def test_unpack_frames_clips_the_tail_of_a_ranged_read(cuda, clip):
    """K2 with CvFrameDesc.tail_clip / CvStreamDesc.tail_clip: the last frame of a range that stops short of its block's end is
    validated as the whole frame the worker sent, but only data_len - tail_clip payload bytes are copied; bytes behind the range stay
    untouched.  (The reference trims such a chunk on the host: fs_reader_buffer.rs:283-301, reader.rs:71-81.)"""
    import torch
    from curvine_b200 import kernels as K
    blocks = [_rand(3 * 4096 + 1234, 70), _rand(4096, 71)]
    wire, descs, streams, total = _build_wire(blocks, 4096, [900, 901], 1)
    last0 = max(i for i, d in enumerate(descs) if d.block == 0)
    c = min(clip, descs[last0].data_len)
    descs[last0].tail_clip = c
    streams[0].tail_clip = c
    want = bytearray(b"\xEE" * (total + 32))
    off = 0
    for bi, b in enumerate(blocks):
        n = len(b) - (c if bi == 0 else 0)
        want[off:off + n] = b.tobytes()[:n]
        off += len(b)
    dst = torch.full((total + 32,), 0xEE, dtype=torch.uint8, device=cuda)
    crc, err = K.unpack_frames(_to_dev(wire, cuda), K.frame_descs_to_device(descs, cuda), len(descs), 2, dst, 1, total)
    assert (K.u32(err) == 0).all()
    assert dst.cpu().numpy().tobytes() == bytes(want)
    assert K.u32(crc).tolist() == [clib.crc(1, blocks[0][:len(blocks[0]) - c]), clib.crc(1, blocks[1])]
    exp = K.expand_streams(K.stream_descs_to_device(streams, cuda), len(streams), len(descs), cuda)
    assert exp.cpu().numpy().tobytes() == K.frame_descs_to_device(descs, cuda).cpu().numpy().tobytes()


def test_unpack_frames_flags_bad_prefixes(cuda):
    import torch
    from curvine_b200 import kernels as K
    from curvine_b200 import _lib as L
    blocks = [_rand(8192, 1)]
    wire, descs, _, total = _build_wire(blocks, 4096, [77], 0)
    # frame 1 becomes an error response (status 0x13, KAT 19) with wrong seq
    off = descs[1].wire_off
    wire[off + 9] = 19
    wire[off + 21] ^= 0x40
    dst = torch.zeros(total, dtype=torch.uint8, device=cuda)
    _, err = K.unpack_frames(_to_dev(wire, cuda), K.frame_descs_to_device(descs, cuda), 2, 1, dst, 0, total)
    e = K.u32(err)
    assert e[0] == 0 and e[1] == (0x08 | 0x20)


@pytest.mark.parametrize("poly", [0, 1])
def test_pack_then_unpack_is_identity(cuda, poly):
    """K4 -> K2 loop-back: pack(payload) gives the oracle's wire bytes; unpack(pack(x)) == x; CRCs agree."""
    import torch
    from curvine_b200 import kernels as K
    blocks = [_rand(n, 40 + i) for i, n in enumerate([300000, 131072, 5])]
    chunk = 65536
    wire, descs, _, total = _build_wire(blocks, chunk, [-5, 6, 7], poly)
    src = _to_dev(np.concatenate(blocks), cuda)
    d_desc = K.frame_descs_to_device(descs, cuda)
    d_wire = torch.zeros(len(wire), dtype=torch.uint8, device=cuda)
    crc_src = K.pack_frames(src, d_desc, len(descs), len(blocks), d_wire, poly, total)
    assert d_wire.cpu().numpy().tobytes() == wire.tobytes()
    dst = torch.zeros(total, dtype=torch.uint8, device=cuda)
    crc_dst, err = K.unpack_frames(d_wire, d_desc, len(descs), len(blocks), dst, poly, total)
    assert torch.equal(dst, src) and (K.u32(err) == 0).all()
    assert K.u32(crc_src).tolist() == K.u32(crc_dst).tolist() == [clib.crc(poly, b) for b in blocks]


def test_gather_pages(cuda):
    """K3: arbitrary (src_off, len, dst_off) segments, every alignment combination."""
    import torch
    from curvine_b200 import kernels as K
    rng = np.random.default_rng(3)
    src = _rand(3 << 20, 8)
    segs, pos = [], 0
    for i in range(200):
        n = int(rng.choice([0, 1, 15, 16, 17, 4096, 4097, 131072, 262144 + 3]))
        so = int(rng.integers(0, len(src) - n))
        segs.append((so, pos, n))
        pos += n + int(rng.integers(0, 5))
    want = np.zeros(pos + 16, dtype=np.uint8)
    for so, do, n in segs:
        want[do:do + n] = src[so:so + n]
    dst = torch.zeros(pos + 16, dtype=torch.uint8, device=cuda)
    K.gather_pages(_to_dev(src, cuda), K.segs_to_device(segs, cuda), len(segs), sum(s[2] for s in segs), dst)
    assert dst.cpu().numpy().tobytes() == want.tobytes()


@pytest.mark.parametrize("n_segs", [4095, 4096, 4097, 13001])
def test_many_small_pieces_multi_tile_scan(cuda, n_segs):
    """More pieces than one scan tile (4096): FUSE-shaped scatter of thousands of tiny pages, and the CRC of
    thousands of small blocks -- the prefix sum over piece unit counts spans several tiles, zero-length pieces included."""
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


@pytest.mark.parametrize("world", [2, 8])
def test_deinterleave_blocks(cuda, world):
    import torch
    from curvine_b200 import kernels as K
    bs, nb = 65536, 37
    file_len = bs * nb - 1000
    data = _rand(file_len, 21)
    per = (nb + world - 1) // world
    stride = per * bs
    gathered = np.zeros(world * stride, dtype=np.uint8)
    for b in range(nb):
        blk = data[b * bs:(b + 1) * bs]
        o = (b % world) * stride + (b // world) * bs
        gathered[o:o + len(blk)] = blk
    dst = torch.zeros(file_len, dtype=torch.uint8, device=cuda)
    K.deinterleave_blocks(_to_dev(gathered, cuda), stride, world, bs, nb, file_len, dst)
    assert dst.cpu().numpy().tobytes() == data.tobytes()


def test_crc_hypothesis_random_buffers(cuda):
    """SURVEY §7 parity test 7: GPU == zlib.crc32 (== crc32fast) and == CRC-32C oracle on generated buffers,
    lengths and base alignments drawn by hypothesis."""
    from hypothesis import given, settings, strategies as st
    from curvine_b200 import kernels as K
    big = _rand(3 << 20, 77)
    d_big = _to_dev(big, cuda)

    @settings(max_examples=40, deadline=None)
    @given(st.lists(st.tuples(st.integers(0, (3 << 20) - 1), st.integers(0, 300000)), min_size=1, max_size=12), st.integers(0, 1))
    def run(spans, poly):
        offs = [o for o, _ in spans]
        lens = [min(n, len(big) - o) for o, n in spans]
        got = K.u32(K.crc_blocks(d_big, offs, lens, poly))
        for g, o, n in zip(got, offs, lens):
            assert int(g) == clib.crc(poly, big[o:o + n])
            if poly == 0:
                assert int(g) == zlib.crc32(big[o:o + n].tobytes())

    run()


@pytest.mark.parametrize("world", [2, 8])
def test_gather_shards_p2p_local_pointers(cuda, world):
    """The fused gather reads each block from its owner's shard pointer (here all local) into file order."""
    import torch
    from curvine_b200 import kernels as K
    bs, nb = 65536, 37
    file_len = bs * nb - 1000
    data = _rand(file_len, 31)
    per = (nb + world - 1) // world
    shards = [torch.zeros(per * bs + 16 * g, dtype=torch.uint8, device=cuda) for g in range(world)]  # separate allocations
    for b in range(nb):
        blk = data[b * bs:(b + 1) * bs]
        shards[b % world][(b // world) * bs:(b // world) * bs + len(blk)] = _to_dev(blk, cuda)
    dst = torch.zeros(file_len, dtype=torch.uint8, device=cuda)
    K.gather_shards_p2p([s.data_ptr() for s in shards], bs, nb, file_len, dst)
    assert dst.cpu().numpy().tobytes() == data.tobytes()


def test_unpack_rejects_oversized_and_negative_frames(cuda):
    """decode_protocol limits (rpc_message.rs:329-334): data_len < 0 and > 16 MiB are flagged by K2's prefix check."""
    import struct
    import torch
    from curvine_b200 import kernels as K
    from curvine_b200._lib import CvFrameDesc
    payload = _rand(4096, 3)
    good = W.encode(W.success(W.request(81, W.REQ_RUNNING, 9, 1), b"", payload.tobytes()))
    too_big = bytearray(good)
    too_big[0:4] = struct.pack(">i", 18 + (16 << 20) + 1)
    negative = bytearray(good)
    negative[0:4] = struct.pack(">i", 17)
    wire = np.frombuffer(bytes(good) + bytes(too_big) + bytes(negative), dtype=np.uint8).copy()
    descs = [CvFrameDesc(i * len(good), i * 4096, 4096, 0, 9, 1, 0, 81, 0x03) for i in range(3)]
    dst = torch.zeros(3 * 4096, dtype=torch.uint8, device=cuda)
    _, err = K.unpack_frames(_to_dev(wire, cuda), K.frame_descs_to_device(descs, cuda), 3, 1, dst, 0, 3 * 4096)
    e = K.u32(err)
    assert e[0] == 0 and e[1] & 0x40 and e[1] & 0x01 and e[2] & 0x40 and e[2] & 0x01
