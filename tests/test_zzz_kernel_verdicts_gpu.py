"""The kernels' verdicts -- the outputs that decide whether delivered bytes are accepted -- against a plain restatement, field by field.

  * K2's prefix validation (prep_unpack_kernel): one CV_FERR_* bit per field of every received frame.  A stream of good frames over
    several blocks, at rotating wire and destination phases, is copied with exactly one frame differing from its descriptor in exactly
    one prefix field (req_id, code, status, seq_id, header_len, total_len, the data length total_len implies).  err_flags must equal the
    restatement of decode_protocol + check_response (rpc_message.rs:320-334, raw_client.rs:100-116) over the oracle's wire bytes bit for
    bit; every unflagged frame's payload must land as the oracle decodes it; every block without a flagged frame must carry the oracle's
    CRC; and nothing may depend on which of d_block_crc / d_err_flags is NULL.  A frame of exactly 16 MiB is legal.
  * K2 with a protobuf header in front of the payload (CvFrameDesc.header_len 1, 7, 300) at every destination phase and tail_clip.
  * cvk_verify_crcs / cvk_verify_crcs_masked: one count per mismatching entry (not per warp), accumulated into d_n_bad; the mask is 0
    on skipped entries; both at sizes around the warp and CTA edges.
  * The launchers' argument contracts: a poly other than 0 / 1, empty inputs, interleave geometry that cannot be walked, and blocks
    that lie wholly past file_len.

Outputs are guard-filled, so a verdict the kernel never wrote shows.  Runs on the host-side stand-ins too (tests/simt_emu);
tests/test_kernel_verdicts_mutants.py checks there that planted bugs in these verdicts fail the tests aimed at them."""
import ctypes
import struct

import numpy as np
import pytest

from curvine_b200 import _lib
from oracle import clib, wire as W
from test_kernels_gpu import _rand, _to_dev

pytestmark = pytest.mark.gpu

# include/curvine_b200_kernels.h
TOTAL_LEN, HEADER_LEN, CODE, STATUS, REQ_ID, SEQ_ID, DATA_RANGE = 0x01, 0x02, 0x04, 0x08, 0x10, 0x20, 0x40
INVALID_VALUE = 1  # cudaErrorInvalidValue
RUNNING_OK = W.status_encode(W.REQ_RUNNING, W.RESP_SUCCESS)  # 0x03

PREFIX = struct.Struct(">iiBBqi")  # total_len, header_len, code, status, req_id, seq_id
GUARD = 0xEE
GUARD32 = 0x5A5A5A5A
SLACK = 64  # the walkers may read the rest of a source's last 16-byte granule
REQ_IDS = [0x0123456789ABCDEF, -5, 1 << 40, 77]  # high words set and clear, and a negative id


def _torch():
    import torch
    return torch


def _K():
    from curvine_b200 import kernels as K
    return K


def _sync():
    _torch().cuda.synchronize()


def _p(t):
    return _K()._ptr(t)


def _guarded(n, cuda, value=GUARD):
    torch = _torch()
    return torch.full((n,), value, dtype=torch.uint8, device=cuda)


def _guarded32(n, cuda):
    torch = _torch()
    return torch.full((n,), GUARD32, dtype=torch.int32, device=cuda)


def _s64(v):
    return (v + (1 << 63)) % (1 << 64) - (1 << 63)


# ---- the restatement


def _verdict(prefix, d):
    """CV_FERR_* bits of one received 22-byte prefix against its frame descriptor: decode_protocol's data-length limits, then
    check_response's echoes and the lengths the descriptor expects, each field on its own"""
    total, hsz, code, status, req_id, seq_id = PREFIX.unpack(bytes(prefix))
    e = 0
    try:
        W.decode_protocol(bytes(prefix))
    except W.WireError:
        e |= DATA_RANGE
    if total != W.HEAD_SIZE + d.header_len + d.data_len:
        e |= TOTAL_LEN
    if hsz != d.header_len:
        e |= HEADER_LEN
    if code != d.code:
        e |= CODE
    if status != d.status:
        e |= STATUS
    if req_id != d.req_id:
        e |= REQ_ID
    if seq_id != d.seq_id:
        e |= SEQ_ID
    return e


def _payload(wire, d):
    """the payload the oracle decodes from the frame at d.wire_off (None when the oracle rejects its prefix)"""
    end = d.wire_off + W.PROTOCOL_SIZE + d.header_len + d.data_len
    try:
        msgs, used = W.decode_stream(wire[d.wire_off:end].tobytes())
    except W.WireError:
        return None
    assert used == end - d.wire_off and len(msgs) == 1 and len(msgs[0].header) == d.header_len
    return np.frombuffer(msgs[0].data, dtype=np.uint8)


# ---- a stream of good frames


def _stream(lens, heads, seed, per_block=3, dst_phase=lambda i: (7 * i + i // 2) % 16, clips=None):
    """Good Running frames as the worker sends them, `per_block` to a block, each block with its own request id.  A gap in front of
    every frame puts frame i's payload at wire phase 5i mod 16, and a gap of at least 16 guard bytes in front of every destination
    puts it at dst_phase(i).  Headers are random bytes, so a payload taken from the wrong place shows.
    -> (wire with SLACK bytes behind it, [CvFrameDesc], number of blocks, destination length)"""
    from curvine_b200._lib import CvFrameDesc
    rng = np.random.default_rng(seed)
    wire, descs, dpos = bytearray(), [], 0
    for i, (n, h) in enumerate(zip(lens, heads)):
        b, seq = i // per_block, i % per_block + 1
        rid = REQ_IDS[b % len(REQ_IDS)]
        wire += bytes((5 * i - len(wire) - W.PROTOCOL_SIZE - h) % 16)
        dpos += 16 + (dst_phase(i) - dpos - 16) % 16
        header = rng.integers(0, 256, size=h, dtype=np.uint8).tobytes()
        data = rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()
        d = CvFrameDesc(len(wire), dpos, n, h, rid, seq, b, W.RPC_CODE_READ_BLOCK, RUNNING_OK)
        d.tail_clip = clips[i] if clips else 0
        descs.append(d)
        wire += W.encode(W.success(W.request(W.RPC_CODE_READ_BLOCK, W.REQ_RUNNING, rid, seq), header, data))
        dpos += n
    return np.frombuffer(bytes(wire) + bytes(SLACK), dtype=np.uint8).copy(), descs, descs[-1].block + 1, dpos + SLACK


def _unpack(cuda, d_wire, d_desc, n_frames, n_blocks, dst_len, poly, total, want_crc, want_err):
    """cvk_unpack_frames into a guard-filled destination and guard-filled CRC and flag outputs (or NULL) -> (bytes, CRCs, flags)"""
    K = _K()
    dst = _guarded(dst_len, cuda)
    crc = _guarded32(n_blocks, cuda) if want_crc else None
    err = _guarded32(n_frames, cuda) if want_err else None
    _lib.check(_lib.lib().cvk_unpack_frames(_p(d_wire), _p(d_desc), n_frames, n_blocks, _p(dst), poly, total, _p(crc), _p(err),
                                            K._stream_ptr()), "cvk_unpack_frames")
    _sync()
    return dst.cpu().numpy(), None if crc is None else K.u32(crc).tolist(), None if err is None else K.u32(err).tolist()


def _check_k2(cuda, wire, descs, n_blocks, dst_len, poly, what=""):
    """K2 with both outputs, without the CRCs and without the flags.  Asserts the restated flags bit for bit, the oracle's payload of
    every unflagged frame (up to its tail_clip), guard bytes everywhere else but inside flagged frames' destinations, the oracle's CRC
    of every block without a flagged frame, and the same bytes, flags and CRCs whichever output is NULL -> the flags"""
    K = _K()
    want = [_verdict(wire[d.wire_off:d.wire_off + W.PROTOCOL_SIZE], d) for d in descs]
    d_wire, d_desc = _to_dev(wire, cuda), K.frame_descs_to_device(descs, cuda)
    total = sum(d.data_len for d in descs)
    runs = {(c, e): _unpack(cuda, d_wire, d_desc, len(descs), n_blocks, dst_len, poly, total, c, e) for c, e in ((1, 1), (0, 1), (1, 0))}
    for (c, e), (_, _, err) in runs.items():
        if e:
            bad = [(i, hex(g), hex(w)) for i, (g, w) in enumerate(zip(err, want)) if g != w]
            assert not bad, (what, "crc" if c else "no crc", "frame, flags, restated", bad)
    expect, free = np.full(dst_len, GUARD, dtype=np.uint8), np.zeros(dst_len, dtype=bool)
    delivered = {}
    for i, d in enumerate(descs):
        n = d.data_len - min(d.tail_clip, d.data_len)
        if want[i]:
            free[d.dst_off:d.dst_off + n] = True  # a rejected frame's bytes are the caller's to discard
            continue
        data = _payload(wire, d)
        assert data is not None, (what, i)
        expect[d.dst_off:d.dst_off + n] = data[:n]
        delivered.setdefault(d.block, []).append(data[:n])
    for (c, e), (dst, _, _) in runs.items():
        wrong = np.nonzero((dst != expect) & ~free)[0]
        assert not wrong.size, (what, "crc" if c else "no crc", "flags" if e else "no flags", "wrong bytes at", wrong[:16].tolist())
    assert np.array_equal(runs[1, 1][0], runs[0, 1][0]) and np.array_equal(runs[1, 1][0], runs[1, 0][0]), what
    flagged = {d.block for d, f in zip(descs, want) if f}
    crc, crc_no_err = runs[1, 1][1], runs[1, 0][1]
    assert crc == crc_no_err, what
    for b in range(n_blocks):
        if b not in flagged:
            assert crc[b] == clib.crc(poly, np.concatenate(delivered.get(b, [np.zeros(0, np.uint8)]))), (what, "block", b)
    return want


# ---- (a) one field at a time

LENS = [1, 15, 16, 17, 31, 511, 512, 513, 4095, 4096, 4097, 8191, 20000, 33, 3, 70000]
HEADS = [7 if i % 5 == 2 else 0 for i in range(len(LENS))]  # three frames carry a header


def _variants(field):
    """[(label, which frames it applies to: with a header / without / any, new value of `field` from the good prefix's fields)]"""
    with_h, without_h, any_h = True, False, None
    if field == "req_id":  # the high word, the low word, the sign bit on their own
        return [("req_id ^ %#x" % m, any_h, lambda p, m=m: _s64(p["req_id"] ^ m)) for m in (1 << 32, 1 << 47, 1 << 62, 1, 1 << 31, 1 << 63)]
    if field == "code":  # every other value of the low nibble, then of the high nibble
        return [("code ^ %#x" % m, any_h, lambda p, m=m: p["code"] ^ m) for m in list(range(1, 16)) + [k << 4 for k in range(1, 16)]]
    if field == "status":  # every bit flipped; flipping bit 4 of 0x03 gives 0x13, the error response to a Running request
        return [("status ^ %#x" % (1 << k), any_h, lambda p, k=k: p["status"] ^ (1 << k)) for k in range(8)]
    if field == "seq_id":
        return [("seq_id + 1", any_h, lambda p: p["seq_id"] + 1), ("seq_id - 1", any_h, lambda p: p["seq_id"] - 1),
                ("INIT_SEQ_ID", any_h, lambda p: W.INIT_SEQ_ID), ("END_SEQ_ID", any_h, lambda p: W.END_SEQ_ID)]
    if field == "header_len":  # total_len still what the descriptor expects: only the split between header and data moves
        return [("a 5-byte header where none is expected", without_h, lambda p: 5), ("header_len -1", without_h, lambda p: -1),
                ("header_len -2^31", without_h, lambda p: -(1 << 31)), ("the header missing", with_h, lambda p: 0),
                ("header_len -1 instead of 7", with_h, lambda p: -1), ("header_len + 1", with_h, lambda p: p["header_len"] + 1)]
    if field == "total_len":
        return [("total_len %+d" % s, any_h, lambda p, s=s: p["total_len"] + s) for s in (1, -1, 1, -1, 1, -1)]
    if field == "data_len":  # through total_len: a data length of exactly 16 MiB is legal (only the descriptor disagrees)
        return [("data exactly 16 MiB", any_h, lambda p: W.HEAD_SIZE + p["header_len"] + W.MAX_DATA_SIZE),
                ("data 16 MiB + 1", any_h, lambda p: W.HEAD_SIZE + p["header_len"] + W.MAX_DATA_SIZE + 1),
                ("data -1", any_h, lambda p: W.HEAD_SIZE + p["header_len"] - 1),
                ("total_len -1", any_h, lambda p: -1), ("total_len 2^31 - 1", any_h, lambda p: (1 << 31) - 1)]
    raise ValueError(field)


FIELDS = ["req_id", "code", "status", "seq_id", "header_len", "total_len", "data_len"]


@pytest.mark.parametrize("poly", [0, 1])
@pytest.mark.parametrize("field", FIELDS)
def test_k2_flags_one_field_at_a_time(cuda, field, poly):
    """Copies of a good stream in which exactly one frame's prefix differs from its descriptor in exactly one field: the flags of
    every frame equal the restatement bit for bit, and the frame that differs is flagged."""
    wire, descs, n_blocks, dst_len = _stream(LENS, HEADS, 100 + poly)
    assert _check_k2(cuda, wire, descs, n_blocks, dst_len, poly, "good stream") == [0] * len(descs)
    names = ("total_len", "header_len", "code", "status", "req_id", "seq_id")
    for k, (label, header, change) in enumerate(_variants(field)):
        pick = [i for i, h in enumerate(HEADS) if header is None or (h > 0) == header]
        f = pick[(5 * k + poly) % len(pick)]
        off = descs[f].wire_off
        p = dict(zip(names, PREFIX.unpack(wire[off:off + W.PROTOCOL_SIZE].tobytes())))
        p[field if field != "data_len" else "total_len"] = change(p)
        bad = wire.copy()
        bad[off:off + W.PROTOCOL_SIZE] = np.frombuffer(PREFIX.pack(*(p[x] for x in names)), dtype=np.uint8)
        flags = _check_k2(cuda, bad, descs, n_blocks, dst_len, poly, (label, "frame", f))
        assert flags[f] and not any(flags[:f] + flags[f + 1:]), (label, f, flags)


@pytest.mark.parametrize("poly", [0, 1])
def test_k2_accepts_a_frame_of_exactly_16_mib(cuda, poly):
    """CV_MAX_DATA_SIZE is the largest legal payload (decode_protocol rejects only more): a 16 MiB frame is delivered with flags 0, its
    bytes and CRC exact; a real frame of 16 MiB + 1 behind it, whose descriptor expects exactly that, is flagged for its data range
    alone; a small frame behind both is delivered."""
    wire, descs, n_blocks, dst_len = _stream([W.MAX_DATA_SIZE, W.MAX_DATA_SIZE + 1, 4097], [0, 0, 0], 160 + poly, per_block=1)
    assert _check_k2(cuda, wire, descs, n_blocks, dst_len, poly) == [0, DATA_RANGE, 0]


# ---- (b) a payload behind a header


@pytest.mark.parametrize("h", [1, 7, 300])
def test_k2_takes_the_payload_from_behind_the_header(cuda, h):
    """Frames with an h-byte header (CvFrameDesc.header_len = h): the payload starts h bytes behind the prefix.  32 frames, destination
    phases 0..15 twice over against rotating wire phases, tail_clip from 0 to the whole payload; both polys, every output combination."""
    lens = [1, 2, 15, 16, 17, 100, 511, 512, 513, 4095, 4096, 4097, 9000, 65539, 31, 33] * 2
    clips = [[0, 1, 15, 16, 17, 511, n - 1, n][i % 8] for i, n in enumerate(lens)]
    clips = [min(c, n) for c, n in zip(clips, lens)]
    wire, descs, n_blocks, dst_len = _stream(lens, [h] * len(lens), 200 + h, per_block=4, dst_phase=lambda i: i % 16, clips=clips)
    for poly in (0, 1):
        assert _check_k2(cuda, wire, descs, n_blocks, dst_len, poly, (h, poly)) == [0] * len(descs)


# ---- (c) cvk_verify_crcs / cvk_verify_crcs_masked

VERIFY_SIZES = [1, 31, 32, 33, 255, 256, 257, 1000003]
N_BAD_START = 12345  # d_n_bad is added to, never set


def _mismatch_sets(n, rng):
    i = np.arange(n)
    warps = (n + 31) // 32
    return {"none": np.zeros(n, dtype=bool), "all": np.ones(n, dtype=bool), "every lane of one warp": i // 32 == warps // 2,
            "one per warp": i % 32 == (i // 32 * 7) % 32, "random": rng.random(n) < 0.37}


def _verify_inputs(n, bad, rng):
    """CRCs and expected values that differ in one bit (rotating through all 32) exactly where `bad` says"""
    crc = rng.integers(0, 1 << 32, size=n, dtype=np.uint64).astype(np.uint32)
    expect = crc ^ (bad.astype(np.uint32) << (np.arange(n) % 32).astype(np.uint32))
    return crc, expect


def _run_verify(cuda, crc, expect, skip, masked, with_mask):
    """cvk_verify_crcs (masked=False) or cvk_verify_crcs_masked, twice on the same input -> (d_n_bad, mask or None)"""
    torch, K = _torch(), _K()
    n = len(crc)
    d_crc, d_exp = (torch.from_numpy(a.view(np.int32)).to(cuda) for a in (crc, expect))
    d_skip = None if skip is None else _to_dev(skip, cuda)
    n_bad = torch.full((1,), N_BAD_START, dtype=torch.int32, device=cuda)
    mask = _guarded(n + SLACK, cuda) if with_mask else None
    L = _lib.lib()
    for _ in range(2):
        if masked:
            rc = L.cvk_verify_crcs_masked(_p(d_crc), _p(d_exp), _p(d_skip), n, _p(n_bad), _p(mask), K._stream_ptr())
        else:
            rc = L.cvk_verify_crcs(_p(d_crc), _p(d_exp), n, _p(n_bad), _p(mask), K._stream_ptr())
        _lib.check(rc, "cvk_verify_crcs" + ("_masked" if masked else ""))
    _sync()
    return int(n_bad.item()), None if mask is None else mask.cpu().numpy()


def _check_verify(got, want, what):
    """two calls' worth of counts on top of N_BAD_START, and the mask (when there is one) = want, guard bytes behind it"""
    n_bad, mask = got
    assert n_bad == N_BAD_START + 2 * int(want.sum()), (what, n_bad - N_BAD_START, 2 * int(want.sum()))
    if mask is not None:
        n = len(want)
        assert np.array_equal(mask[:n], want.astype(np.uint8)), (what, np.nonzero(mask[:n] != want)[0][:16].tolist())
        assert (mask[n:] == GUARD).all(), what


@pytest.mark.parametrize("n", VERIFY_SIZES)
def test_verify_crcs_counts_every_mismatch(cuda, n):
    """d_n_bad += the number of mismatching ENTRIES (a warp with 32 mismatches adds 32), over two calls; d_bad_mask[i] = mismatch,
    nothing behind n; the mask is optional.  cvk_verify_crcs and cvk_verify_crcs_masked without a skip mask agree."""
    rng = np.random.default_rng(n)
    for name, bad in _mismatch_sets(n, rng).items():
        crc, expect = _verify_inputs(n, bad, rng)
        for masked in (False, True):
            for with_mask in (True, False):
                _check_verify(_run_verify(cuda, crc, expect, None, masked, with_mask), bad, (name, masked, with_mask))


@pytest.mark.parametrize("n", VERIFY_SIZES)
def test_verify_crcs_masked_leaves_skipped_entries_out(cuda, n):
    """cvk_verify_crcs_masked: an entry whose d_skip byte is non-zero (any value) is neither counted nor marked -- its mask byte is 0
    -- whatever its CRCs; skip masks of zeros, all, random, and exactly the mismatches, against every mismatch set."""
    rng = np.random.default_rng(1000 + n)
    for name, bad in _mismatch_sets(n, rng).items():
        crc, expect = _verify_inputs(n, bad, rng)
        marks = rng.integers(1, 256, size=n, dtype=np.uint8)  # "skip" is any non-zero byte
        skips = {"zeros": np.zeros(n, dtype=bool), "all": np.ones(n, dtype=bool), "random": rng.random(n) < 0.5, "the mismatches": bad}
        for sname, sk in skips.items():
            skip = np.where(sk, marks, 0).astype(np.uint8)
            for with_mask in (True, False):
                _check_verify(_run_verify(cuda, crc, expect, skip, True, with_mask), bad & ~sk, (name, sname, with_mask))


# ---- (d) argument contracts of the launchers


def _untouched(bufs):
    _sync()
    for name, t, value in bufs:
        a = t.cpu().numpy()
        assert (a == value).all(), (name, np.nonzero(a != value)[0][:16].tolist())


def test_a_poly_other_than_0_or_1_is_refused_before_anything_runs(cuda):
    """cvk_crc_blocks, cvk_unpack_frames and cvk_pack_frames return cudaErrorInvalidValue for a poly other than 0 / 1, launch nothing
    and write nothing; the same inputs with poly 0 and 1 give the oracle's results."""
    torch, K = _torch(), _K()
    L, s = _lib.lib(), K._stream_ptr()
    wire, descs, n_blocks, dst_len = _stream([5000, 17], [0, 0], 7, per_block=2)
    d_wire, d_desc = _to_dev(wire, cuda), K.frame_descs_to_device(descs, cuda)
    payload = np.concatenate([_payload(wire, d) for d in descs])
    image = np.zeros(dst_len, dtype=np.uint8)  # K4 reads frame f's payload at d_src + dst_off, as K2 delivers it
    for d in descs:
        image[d.dst_off:d.dst_off + d.data_len] = _payload(wire, d)
    src = _to_dev(image, cuda)
    offs = torch.tensor([descs[0].dst_off, descs[0].dst_off + 3], dtype=torch.int64, device=cuda)
    lens = torch.tensor([descs[0].data_len, 100], dtype=torch.int64, device=cuda)
    dst, out_wire, crc, err = _guarded(dst_len, cuda), _guarded(len(wire), cuda), _guarded32(2, cuda), _guarded32(2, cuda)
    total = len(payload)
    for poly in (2, 3, -1, 255, 1 << 30):
        before = K.launch_count()
        assert L.cvk_crc_blocks(_p(src), _p(offs), _p(lens), 2, poly, descs[0].data_len + 100, _p(crc), s) == INVALID_VALUE, poly
        assert L.cvk_unpack_frames(_p(d_wire), _p(d_desc), 2, 1, _p(dst), poly, total, _p(crc), _p(err), s) == INVALID_VALUE, poly
        assert L.cvk_pack_frames(_p(src), _p(d_desc), 2, 1, _p(out_wire), poly, total, _p(crc), s) == INVALID_VALUE, poly
        assert K.launch_count() == before, poly
    _untouched([("dst", dst, GUARD), ("wire", out_wire, GUARD), ("crc", crc, GUARD32), ("flags", err, GUARD32)])
    for poly in (0, 1):
        _lib.check(L.cvk_crc_blocks(_p(src), _p(offs), _p(lens), 2, poly, descs[0].data_len + 100, _p(crc), s))
        _sync()
        assert K.u32(crc).tolist() == [clib.crc(poly, payload[:descs[0].data_len]), clib.crc(poly, payload[3:103])]
        assert _check_k2(cuda, wire, descs, n_blocks, dst_len, poly) == [0, 0]
        _lib.check(L.cvk_pack_frames(_p(src), _p(d_desc), 2, 1, _p(out_wire), poly, total, _p(crc), s))
        _sync()
        assert K.u32(crc).tolist()[0] == clib.crc(poly, payload)
        got = out_wire.cpu().numpy()
        assert all(np.array_equal(got[d.wire_off:d.wire_off + W.PROTOCOL_SIZE + d.data_len],
                                  wire[d.wire_off:d.wire_off + W.PROTOCOL_SIZE + d.data_len]) for d in descs)


def test_empty_inputs_launch_nothing_and_write_nothing(cuda):
    """n == 0 returns 0 from every launcher with no launch and no output byte written; so does K5 with total_elems == 0 over a non-empty
    table, and K3-strided over descriptors whose rows are all empty."""
    torch, K = _torch(), _K()
    L, s = _lib.lib(), K._stream_ptr()
    src = _to_dev(_rand(4096 + SLACK, 9), cuda)
    dst, mask, wire = _guarded(4096, cuda), _guarded(256, cuda), _guarded(4096, cuda)
    out32, n_bad = _guarded32(64, cuda), _guarded32(1, cuda)
    c32 = torch.arange(64, dtype=torch.int32, device=cuda)
    zeros64 = torch.zeros(4, dtype=torch.int64, device=cuda)
    _, descs, _, _ = _stream([100], [0], 3, per_block=1)
    d_desc = K.frame_descs_to_device(descs, cuda)
    from curvine_b200._lib import CvStreamDesc
    d_streams = K.stream_descs_to_device([CvStreamDesc(0, 0, 100, 1, 64, 1, 0, 0, 81, 3)], cuda)
    d_segs = K.segs_to_device([(0, 0, 100)], cuda)
    d_empty_rows = K.strided_segs_to_device([(0, 0, 0, 5, 16, 16), (0, 0, 64, 0, 64, 64)], cuda)
    d_cast, _ = K.cast_segs_to_device([(0, 0, 64, 2, 256, 256, _lib.DTYPE_F32, _lib.DTYPE_BF16)], cuda)
    d_scales = K.scale_segs_to_device([None], cuda)
    shard_ptrs = (ctypes.c_uint64 * 2)(src.data_ptr(), src.data_ptr())
    calls = {
        "cvk_crc_blocks": lambda: L.cvk_crc_blocks(_p(src), _p(zeros64), _p(zeros64), 0, 0, 0, _p(out32), s),
        "cvk_verify_crcs": lambda: L.cvk_verify_crcs(_p(c32), _p(c32), 0, _p(n_bad), _p(mask), s),
        "cvk_verify_crcs_masked": lambda: L.cvk_verify_crcs_masked(_p(c32), _p(c32), _p(mask), 0, _p(n_bad), _p(mask), s),
        "cvk_unpack_frames": lambda: L.cvk_unpack_frames(_p(src), _p(d_desc), 0, 0, _p(dst), 0, 0, _p(out32), _p(out32), s),
        "cvk_pack_frames": lambda: L.cvk_pack_frames(_p(src), _p(d_desc), 0, 0, _p(wire), 1, 0, _p(out32), s),
        "cvk_expand_streams": lambda: L.cvk_expand_streams(_p(d_streams), 0, _p(wire), 0, s),
        "cvk_gather_pages": lambda: L.cvk_gather_pages(_p(src), _p(d_segs), 0, 0, _p(dst), s),
        "cvk_gather_strided": lambda: L.cvk_gather_strided(_p(src), _p(d_segs), 0, 0, _p(dst), s),
        "cvk_gather_strided, empty rows": lambda: L.cvk_gather_strided(_p(src), _p(d_empty_rows), 2, 0, _p(dst), s),
        "cvk_gather_cast": lambda: L.cvk_gather_cast(_p(src), _p(d_cast), 0, 0, _p(dst), s),
        "cvk_gather_cast, total_elems 0": lambda: L.cvk_gather_cast(_p(src), _p(d_cast), 1, 0, _p(dst), s),
        "cvk_gather_cast_scaled": lambda: L.cvk_gather_cast_scaled(_p(src), _p(d_cast), None, 0, 0, _p(dst), s),
        "cvk_gather_cast_scaled, total_elems 0": lambda: L.cvk_gather_cast_scaled(_p(src), _p(d_cast), _p(d_scales), 1, 0, _p(dst), s),
        "cvk_deinterleave_blocks": lambda: L.cvk_deinterleave_blocks(_p(src), 2048, 2, 1024, 0, 4096, _p(dst), s),
        "cvk_gather_shards_p2p": lambda: L.cvk_gather_shards_p2p(shard_ptrs, 2, 1024, 0, 4096, _p(dst), s),
    }
    for name, call in calls.items():
        before = K.launch_count()
        assert call() == 0, name
        assert K.launch_count() == before, name
    _untouched([("dst", dst, GUARD), ("mask", mask, GUARD), ("wire / descriptors", wire, GUARD), ("crc / flags", out32, GUARD32),
                ("n_bad", n_bad, GUARD32)])


def test_interleave_geometry_that_cannot_be_walked_is_refused(cuda):
    """cvk_deinterleave_blocks and cvk_gather_shards_p2p refuse world 0, block_size 0 and 2^31 blocks (and the gather more than 64
    ranks) with cudaErrorInvalidValue, launching nothing and writing nothing."""
    K = _K()
    L, s = _lib.lib(), K._stream_ptr()
    src = _to_dev(_rand(8192 + SLACK, 4), cuda)
    dst = _guarded(8192, cuda)
    ptrs = (ctypes.c_uint64 * 65)(*([src.data_ptr()] * 65))
    before = K.launch_count()
    for world, bs, nb in ((0, 1024, 4), (2, 0, 4), (2, 1024, 1 << 31)):
        assert L.cvk_deinterleave_blocks(_p(src), 4096, world, bs, nb, 4096, _p(dst), s) == INVALID_VALUE, (world, bs, nb)
    for world, bs, nb in ((0, 1024, 4), (65, 1024, 4), (2, 0, 4), (2, 1024, 1 << 31)):
        assert L.cvk_gather_shards_p2p(ptrs, world, bs, nb, 4096, _p(dst), s) == INVALID_VALUE, (world, bs, nb)
    assert K.launch_count() == before
    _untouched([("dst", dst, GUARD)])


@pytest.mark.parametrize("world", [1, 3])
def test_blocks_wholly_past_file_len_are_accepted_and_left_alone(cuda, world):
    """n_blocks may run past the file: blocks that start at or behind file_len are accepted and their destinations keep every byte;
    the block file_len cuts is delivered up to file_len.  Both the de-interleave and the fused shard gather, file_len from 0 up."""
    K = _K()
    bs, nb = 4096 + 5, 10
    data = _rand(nb * bs, 50 + world)
    per = (nb + world - 1) // world
    shards = [np.zeros(per * bs + SLACK, dtype=np.uint8) for _ in range(world)]
    for b in range(nb):
        shards[b % world][(b // world) * bs:(b // world + 1) * bs] = data[b * bs:(b + 1) * bs]
    d_gathered = _to_dev(np.concatenate(shards), cuda)
    d_shards = [_to_dev(x, cuda) for x in shards]
    stride = per * bs + SLACK
    for file_len in (0, 1, 5 * bs, 5 * bs + 1234, nb * bs - 1):
        for how in ("deinterleave", "p2p"):
            dst = _guarded(nb * bs + SLACK, cuda)
            if how == "deinterleave":
                K.deinterleave_blocks(d_gathered, stride, world, bs, nb, file_len, dst)
            else:
                K.gather_shards_p2p([t.data_ptr() for t in d_shards], bs, nb, file_len, dst)
            _sync()
            got = dst.cpu().numpy()
            assert np.array_equal(got[:file_len], data[:file_len]), (how, file_len)
            assert (got[file_len:] == GUARD).all(), (how, file_len, np.nonzero(got[file_len:] != GUARD)[0][:8].tolist())
