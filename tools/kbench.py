"""Kernel-only micro-benchmarks (CUDA events, inputs >> L2): K1 crc, K2 unpack+crc, K3 gather.  Not the bench.py contract."""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from curvine_b200 import _lib, kernels as K  # noqa: E402
from curvine_b200._lib import CvStreamDesc  # noqa: E402


WARM_SEC = 0.25


def timeit(fn, iters=20, warm_sec=None):
    """-> (best ms, median ms).  Warm-up runs the kernel back to back for `warm_sec` of wall time first: the host-side
    setup between cases (Python building descriptor tables) is long enough for the GPU to drop its clocks, and a two-launch
    warm-up then times the ramp instead of the kernel."""
    import time
    warm_sec = WARM_SEC if warm_sec is None else warm_sec
    t0 = time.time()
    fn()
    while time.time() - t0 < warm_sec:
        for _ in range(4):
            fn()
        torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return min(ts), sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=4.0)
    ap.add_argument("--block", type=int, default=4 << 20)
    ap.add_argument("--only", default="")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--seg-shift", type=int, default=0, help="cvk_tune(4, v): segment size 2^v bytes for every launcher (0 = automatic)")
    ap.add_argument("--warm-sec", type=float, default=0.25, help="seconds of back-to-back warm-up launches before timing (0 under ncu)")
    a = ap.parse_args()
    global WARM_SEC
    WARM_SEC = a.warm_sec
    dev = torch.device("cuda:0")
    _lib.check(_lib.lib().cvk_init(0))
    if a.seg_shift:
        _lib.check(_lib.lib().cvk_tune(4, a.seg_shift))
    total = int(a.gib * (1 << 30)) // a.block * a.block
    nb = total // a.block
    data = torch.randint(0, 2 ** 31, (total // 4,), dtype=torch.int32, device=dev).view(torch.uint8)
    offs = torch.arange(nb, dtype=torch.int64, device=dev) * a.block
    lens = torch.full((nb,), a.block, dtype=torch.int64, device=dev)
    out = torch.empty(nb, dtype=torch.int32, device=dev)
    res = {}
    if not a.only or "k1" in a.only:
        for poly in (0, 1):
            best, med = timeit(lambda: K.crc_blocks_raw(data.data_ptr(), offs, lens, nb, poly, total, out), a.iters)
            res["k1_crc_poly%d" % poly] = {"GBps_best": total / best / 1e6, "GBps_med": total / med / 1e6, "ms": best}
        # one block at a time (latency of a single 4 MiB verify)
        best, med = timeit(lambda: K.crc_blocks_raw(data.data_ptr(), offs, lens, 1, 0, a.block, out), a.iters)
        res["k1_single_block"] = {"us": best * 1e3, "GBps": a.block / best / 1e6}
    if not a.only or "k2" in a.only:
        for chunk in (131072, 1 << 20, 4 << 20):
            fpb = a.block // chunk
            stride = a.block + 22 * fpb
            nb2 = min(nb, int((total - 64) // stride))
            streams = (CvStreamDesc * nb2)()
            for b in range(nb2):
                streams[b] = CvStreamDesc(b * stride, b * a.block, a.block, 1000 + b, chunk, 1, b, b * fpb, 81, 3)
            d_streams = K._struct_array_to_device(streams, dev)
            nf = nb2 * fpb
            d_desc = K.expand_streams(d_streams, nb2, nf, dev)
            # build a valid wire image on the device with K4 (pack) from `data`
            wire = torch.empty(nb2 * stride + 64, dtype=torch.uint8, device=dev)
            K.pack_frames(data, d_desc, nf, nb2, wire, 0, nb2 * a.block, want_crc=False)
            dst = torch.empty(nb2 * a.block, dtype=torch.uint8, device=dev)
            crc = torch.empty(nb2, dtype=torch.int32, device=dev)
            err = torch.empty(nf, dtype=torch.int32, device=dev)
            L = _lib.lib()

            def run():
                _lib.check(L.cvk_unpack_frames(ctypes.c_void_p(wire.data_ptr()), ctypes.c_void_p(d_desc.data_ptr()), nf, nb2,
                                               ctypes.c_void_p(dst.data_ptr()), 0, nb2 * a.block,
                                               ctypes.c_void_p(crc.data_ptr()), ctypes.c_void_p(err.data_ptr()),
                                               ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
            best, med = timeit(run, a.iters)
            n = nb2 * a.block
            ok = bool((err == 0).all().item()) and torch.equal(dst, data[:n])
            K.crc_blocks_raw(data.data_ptr(), offs, lens, nb2, 0, n, out)
            ok = ok and torch.equal(out[:nb2], crc)
            res["k2_unpack_chunk%d" % chunk] = {"payload_GBps": n / best / 1e6, "algo_GBps": (2 * n + 22 * nf) / best / 1e6,
                                                "algo_GBps_med": (2 * n + 22 * nf) / med / 1e6, "ms": best, "ok": ok}
            # K4: the worker-side inverse (pack + CRC at source) over the same frames
            wire2 = torch.empty_like(wire)
            crc4 = torch.empty(nb2, dtype=torch.int32, device=dev)

            def run4():
                _lib.check(L.cvk_pack_frames(ctypes.c_void_p(data.data_ptr()), ctypes.c_void_p(d_desc.data_ptr()), nf, nb2,
                                             ctypes.c_void_p(wire2.data_ptr()), 0, nb2 * a.block, ctypes.c_void_p(crc4.data_ptr()),
                                             ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
            best4, med4 = timeit(run4, a.iters)
            ok4 = torch.equal(wire2[:nb2 * stride], wire[:nb2 * stride]) and torch.equal(crc4, crc)
            res["k4_pack_chunk%d" % chunk] = {"payload_GBps": n / best4 / 1e6, "algo_GBps": (2 * n + 22 * nf) / best4 / 1e6,
                                              "algo_GBps_med": (2 * n + 22 * nf) / med4 / 1e6, "ms": best4, "ok": ok4}
            del wire2
            del wire, dst
    if not a.only or "k3" in a.only:
        n = total // 2
        page = 131072
        segs = [(i * page + 6, i * page, page) for i in range(n // page - 1)]
        d_segs = K.segs_to_device(segs, dev)
        dst = torch.empty(n, dtype=torch.uint8, device=dev)
        tb = sum(s[2] for s in segs)
        best, med = timeit(lambda: K.gather_pages(data, d_segs, len(segs), tb, dst), a.iters)
        ok3 = all(torch.equal(dst[d:d + ln], data[s0:s0 + ln]) for s0, d, ln in (segs[0], segs[len(segs) // 2], segs[-1]))
        res["k3_gather_128k_misaligned"] = {"payload_GBps": tb / best / 1e6, "algo_GBps": 2 * tb / best / 1e6, "algo_GBps_med": 2 * tb / med / 1e6, "ms": best, "ok": ok3}
        segs4k = [(i * 4096 + 4096 + 3, i * 4096, 4096) for i in range(min(n // 4096 - 2, 1 << 18))]
        d_segs4k = K.segs_to_device(segs4k, dev)
        tb4 = sum(s[2] for s in segs4k)
        best, med = timeit(lambda: K.gather_pages(data, d_segs4k, len(segs4k), tb4, dst), a.iters)
        res["k3_gather_4k_pages_misaligned"] = {"payload_GBps": tb4 / best / 1e6, "algo_GBps": 2 * tb4 / best / 1e6, "algo_GBps_med": 2 * tb4 / med / 1e6, "ms": best}
        segsa = [(i * page + 4096, i * page, page) for i in range(n // page - 1)]
        d_segsa = K.segs_to_device(segsa, dev)
        best, med = timeit(lambda: K.gather_pages(data, d_segsa, len(segsa), tb, dst), a.iters)
        res["k3_gather_128k_aligned"] = {"payload_GBps": tb / best / 1e6, "algo_GBps": 2 * tb / best / 1e6, "algo_GBps_med": 2 * tb / med / 1e6, "ms": best}
        d2 = torch.empty(n, dtype=torch.uint8, device=dev)
        best, med = timeit(lambda: d2.copy_(data[:n]), a.iters)
        res["torch_copy"] = {"algo_GBps": 2 * n / best / 1e6, "algo_GBps_med": 2 * n / med / 1e6}
        del d2
    res["seg_shift"] = a.seg_shift or "auto"
    res["launches"] = K.launch_count()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
