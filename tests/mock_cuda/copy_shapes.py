"""TEST INFRASTRUCTURE ONLY: the copies the device reader issues, case by case, on the mock runtime.  For every (tier, copy_group,
call) of a fixed matrix one read runs on a fresh file system handle, and the script prints one JSON object: case name -> the mock's
memcpy/registration counter deltas over the read, the reader's device_stats() and the context's arena_stats().  Only deterministic
configurations: registration inline (register_threads = 0) into a cache nothing is evicted from, arena reads after wait_registered(),
the mock's streams synchronous.  MOCK_CUDA_GDS=1 must be set so that the SSD tier goes through the GDS group path."""
import ctypes
import json
import os
import shutil
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from curvine_b200 import _lib  # noqa: E402

_lib.LIB_PATH = os.environ["CV_TEST_MOCK_CUDA_LIB"]
from curvine_b200 import fs as F  # noqa: E402

FIELDS = ["memcpy_calls", "memcpy_bytes", "register_calls", "h2d_bytes", "blocks", "verified", "reg_hits", "reg_misses", "reg_rejected",
          "dma_jobs", "dma_bytes", "gds_bytes"]
BS = 128 << 10
NB = 41
N = (NB - 1) * BS + 5000  # the last block is short
SMALL = 73 * 4096  # read_many's files: three blocks, the last one short but whole pages (a registered group maps block files back to back)
COMMON = 'fetch_threads = 4\nverify_batch = 4\npinned_slots = 12\ngpu_chunk_size = "64KB"\nregister_threads = 0\nregister_cache = "1GB"\n'


def counters():
    a = (ctypes.c_uint64 * 6)()
    _lib.lib().mock_cuda_counters(a)
    return {"memcpy_calls": a[0], "memcpy_bytes": a[1], "register_calls": a[3]}


def calls(r, fs):
    """-> (call name -> function running one read of the reader's file (of the small files for read_many), the buffers they use)."""
    dst = np.zeros(N + 4096, dtype=np.uint8)
    p = dst.ctypes.data
    # one or two small ranges inside every other block: 37 boundary blocks, more than the staging holds at copy_group 1 and 4
    around = [(2 * BS, 3 * BS, p), (12 * BS - 777, BS + 1554, p + 4 * BS)]  # three whole blocks; a partial, a whole and a partial one
    offs = [b * BS + o for b in range(NB) if b not in (2, 3, 4, 11, 12, 13) for o in (100, 60000) if b * BS + o + 1000 <= N]
    small = np.zeros(len(offs) * 1000, dtype=np.uint8)
    ranges = around + [(o, 1000, small.ctypes.data + i * 1000) for i, o in enumerate(offs)]
    pages = np.zeros(N, dtype=np.uint8)

    def ranged():
        r.seek(BS // 2 + 123)
        return r.read_device(p, 20 * BS, 0)

    def fuse():
        scratch = np.zeros(6 * BS, dtype=np.uint8)
        return r.fuse_read_device(3 * BS + 999, 5 * BS + 17, scratch.ctypes.data, pages.ctypes.data, [i * 4096 for i in range(1400)], 1024)

    def many():
        big = np.zeros(6 * SMALL, dtype=np.uint8)
        return fs.read_many_device(["/s%d" % i for i in range(6)], big.ctypes.data, [i * SMALL for i in range(6)], big.size, 0)

    return {
        "whole": lambda: r.read_device(p, N, 0),
        "ranged": ranged,
        "readv": lambda: r.readv_device(ranges, 0),
        "fuse": fuse,
        "sharded": lambda: r.read_device_sharded(1, 3, p, N, 0),
        "read_many": many,
    }, (dst, small, pages)


def run_case(man, conf, arena, call, path="/f"):
    with F.CurvineFileSystem(conf) as fs:
        fs.load_namespace(man)
        if arena:
            fs.preregister()
            fs.wait_registered()
        a0 = fs.arena_stats()
        r = fs.open(path)
        c0 = counters()
        fns, _bufs = calls(r, fs)
        fns[call]()
        r.verify()
        c1 = counters()
        ds, a1 = r.device_stats(), fs.arena_stats()
        r.complete()
    out = {k: c1[k] - c0[k] for k in c0}
    out.update({k: ds[k] for k in ("h2d_bytes", "blocks", "verified", "reg_hits", "reg_misses", "reg_rejected", "gds_bytes")})
    out.update({k: a1[k] - a0[k] for k in ("dma_jobs", "dma_bytes")})
    return [int(out[k]) for k in FIELDS]


def main():
    assert os.environ.get("MOCK_CUDA_GDS") == "1", "set MOCK_CUDA_GDS=1"
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    d = tempfile.mkdtemp(prefix="cvshape", dir=base)
    results = {}
    try:
        arena_w = F.MiniWorker(["[MEM:64MB]" + d + "/a"], extra_worker='mem_arena = true\narena_segment = "8MB"\narena_reuse_delay = "0ms"\n')
        mem_w = F.MiniWorker(["[MEM]" + d + "/m"])
        ssd_w = F.MiniWorker(["[SSD]" + d + "/s"])
        try:
            mans = {}
            for name, w, st in (("arena", arena_w, 0), ("mem", mem_w, 0), ("ssd", ssd_w, 1)):
                m = w.create_file("/f", 9001, N, BS, storage_type=st)
                m += w.create_file("/h", 9002, N, BS, storage_type=st, mode=2, hole_every=5)
                m += "".join(w.create_file("/s%d" % i, 9100 + i, SMALL, BS, storage_type=st) for i in range(6))
                mans[name] = m
            tiers = {
                "arena": (mans["arena"], True, 'zero_copy = true\narena_preregister = ["%s/a"]\narena_register_slice = "2MB"\n' % d),
                "files": (mans["mem"], True, "zero_copy = true\n"),
                "ring": (mans["mem"], True, "zero_copy = false\n"),
                "framed": (mans["mem"], False, "zero_copy = true\n"),
                "ssd": (mans["ssd"], True, 'zero_copy = false\ngds = "on"\n'),
            }
            for tier, (man, sc, extra) in tiers.items():
                for cg in (1, 4):
                    conf = F.client_conf(short_circuit=sc, b200=COMMON + "copy_group = %d\n" % cg + extra)
                    for call in ("whole", "ranged", "readv", "fuse", "sharded", "read_many"):
                        results["%s/cg%d/%s" % (tier, cg, call)] = run_case(man, conf, tier == "arena", call)
                    results["%s/cg%d/hole" % (tier, cg)] = run_case(man, conf, tier == "arena", "whole", path="/h")
        finally:
            arena_w.stop(), mem_w.stop(), ssd_w.stop()
    finally:
        shutil.rmtree(d, ignore_errors=True)
    print(json.dumps({"fields": FIELDS, "cases": results}))


if __name__ == "__main__":
    main()
