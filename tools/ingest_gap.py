#!/usr/bin/env python
"""Where the headline ingest rate stands between the copy engine and the reader pipeline, on one GPU, in one process.

    python tools/ingest_gap.py [--gib 16] [--reps 3]

Three numbers, each in GB/s of host bytes landed in HBM, each printed with the card's name and power limit:
  1 ceiling   back-to-back 32 MiB H2D copies (cvh_h2d_async) on one stream out of a cudaHostAlloc buffer: what the copy engine
              and the link do with pinned pages the driver allocated
  2 arena     the same 32 MiB copies out of the extents of a --gib file in a pinned arena, laid out as bench.py lays it out (same
              worker settings, 256 MiB segments registered once, copies split at segment edges), no RPC, no verify: what the
              platform does with the arena's pages
  3 headline  bench.py's headline read (cv_read_device + cv_verify through the C ABI, bench's client configuration, a never-read
              file every step), with fetch_sec / (fetch threads x wall): how busy the fetch threads were
The gap 1 -> 2 is the platform's; the gap 2 -> 3 is the reader pipeline's.  One JSON line on stdout."""
import argparse
import ctypes
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from curvine_b200 import _lib  # noqa: E402

GROUP = 32 << 20  # one copy group at the bench shape: copy_group 8 x 4 MiB blocks


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().split(",")
        out["power_limit_w"], out["max_sm_mhz"] = float(q[0]), float(q[1])
    except Exception:  # noqa: BLE001  (a missing nvidia-smi leaves the name alone)
        pass
    return out


def timed_copies(L, pieces, stream, reps):
    """pieces: [(d_dst, h_src, n)] enqueued back to back on `stream`, `reps` times -> GB/s of each rep (device-timed)"""
    import torch
    rates = []
    total = sum(n for _, _, n in pieces)
    for _ in range(reps + 1):  # the first pass warms the path up and is not reported
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for d, h, n in pieces:
            _lib.check(L.cvh_h2d_async(ctypes.c_void_p(d), ctypes.c_void_p(h), n, ctypes.c_void_p(stream), None), "cvh_h2d_async")
        b.record()
        b.synchronize()
        rates.append(total / a.elapsed_time(b) / 1e6)
    return rates[1:]


def arena_extents(arena_dir):
    """-> ({segment: (path, bytes)}, [(segment, offset, length)] of every block descriptor under arena_dir)"""
    segs, ext = {}, []
    for root, _, files in os.walk(arena_dir):
        for f in files:
            p = os.path.join(root, f)
            if f.startswith("seg_"):
                segs[int(f[4:])] = (p, os.path.getsize(p))
            elif os.path.getsize(p) < 128:
                t = open(p).read().split()
                if len(t) == 4 and t[0] == "CVARENA1":
                    ext.append((int(t[1]), int(t[2]), int(t[3])))
    return segs, ext


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=16.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    a = ap.parse_args()
    bench.quiet_stdout()
    import torch
    from curvine_b200 import fs as F
    L = _lib.lib()
    sys.argv = [sys.argv[0], "--gib-per-gpu", str(a.gib)]
    args = bench.parse()
    _, world, local, dist = bench.setup_dist(args)
    _lib.check(L.cvk_init(local), "cvk_init")
    shard = int(args.gib_per_gpu * (1 << 30)) // bench.BLOCK * bench.BLOCK
    ncpu = os.cpu_count() or 8
    threads = max(4, min(16, ncpu // 2))
    slots = 2 * args.verify_batch + threads + 8
    out = {"card": card(), "bytes": shard}
    dst = torch.empty(shard, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    d0 = dst.data_ptr()

    # 1: the copy engine out of cudaHostAlloc pages (1 GiB of them, cycled)
    hb = ctypes.c_void_p()
    ring = 1 << 30
    _lib.check(L.cvh_pinned_alloc(ring, ctypes.byref(hb)), "cvh_pinned_alloc")
    try:
        pieces = [(d0 + off, hb.value + off % ring, GROUP) for off in range(0, shard, GROUP)]
        out["ceiling_GBps"] = timed_copies(L, pieces, stream, a.reps)
    finally:
        L.cvh_pinned_free(hb)

    cluster = bench.Cluster(args, 0, world, dist, shard, need_files_tier=False)
    libc = ctypes.CDLL(None, use_errno=True)
    libc.mmap.restype, libc.mmap.argtypes = ctypes.c_void_p, [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_long]
    libc.munmap.argtypes = [ctypes.c_void_p, ctypes.c_size_t]
    maps = {}
    try:
        # 2: the same copies out of a bench-shaped file's arena extents (a mapping of the segments of our own, registered per segment)
        cluster.create("arena", "/gap/copy", 9000, shard)
        segs, ext = arena_extents(os.path.join(cluster.dir, "arena0"))
        assert sum(n for _, _, n in ext) == shard, "the arena holds %d bytes of descriptors, expected %d" % (sum(n for _, _, n in ext), shard)
        for seg, (p, n) in segs.items():
            fd = os.open(p, os.O_RDWR)
            base = libc.mmap(None, n, 0x1 | 0x2, 0x01, fd, 0)  # PROT_READ|PROT_WRITE, MAP_SHARED
            os.close(fd)
            assert base not in (None, ctypes.c_void_p(-1).value), "mmap %s" % p
            _lib.check(L.cvh_host_register(ctypes.c_void_p(base), n), "cvh_host_register")
            maps[seg] = (base, n)
        ext.sort(key=lambda e: (e[0], e[1]))
        pieces, off = [], 0
        for g in range(0, len(ext), GROUP // bench.BLOCK):  # a group's extents: one copy where they are contiguous inside a segment
            run = None
            for seg, eo, n in ext[g:g + GROUP // bench.BLOCK]:
                if run and run[0] == seg and run[1] + run[2] == eo:
                    run[2] += n
                else:
                    if run:
                        pieces.append((d0 + run[3], maps[run[0]][0] + run[1], run[2]))
                    run = [seg, eo, n, off]
                off += n
            pieces.append((d0 + run[3], maps[run[0]][0] + run[1], run[2]))
        out["arena_GBps"] = timed_copies(L, pieces, stream, a.reps)
        out["arena_copies"] = len(pieces)
        cluster.drop("/gap/copy")
        for base, n in maps.values():
            L.cvh_host_unregister(ctypes.c_void_p(base))
            libc.munmap(ctypes.c_void_p(base), n)
        maps = {}

        # 3: the headline read, as bench.py runs it
        fs = F.CurvineFileSystem(bench.client_conf(args, cluster, True, local, threads, slots, 0))
        try:
            fs.preregister()
            fs.wait_registered()
            leg = bench.run_leg("gap", cluster, fs, "arena", args, 0, world, dist, dst, shard, a.steps, 1, True, 9100)
        finally:
            fs.close()
        st = leg["stats"]
        out["headline_GBps"] = [shard / ms / 1e6 for ms in leg["ingest_ms"]]
        out["fetch_threads"] = threads
        out["fetch_busy"] = st["fetch_sec"] / (threads * st["wall_sec"])
        out["last_step_fetch_thread_sec"], out["last_step_wall_sec"] = st["fetch_sec"], st["wall_sec"]
    finally:
        for base, n in maps.values():
            L.cvh_host_unregister(ctypes.c_void_p(base))
            libc.munmap(ctypes.c_void_p(base), n)
        cluster.close()
    bench.emit(out)


if __name__ == "__main__":
    main()
