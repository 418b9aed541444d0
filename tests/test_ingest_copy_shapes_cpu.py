"""The shape of the copies the device reader issues: how many cudaMemcpyAsync calls move how many bytes, how many host ranges get
registered, and what the reader's and the arena's counters say, for a fixed matrix of reads on the mock runtime
(tests/mock_cuda/copy_shapes.py).  The parity suites check bytes and CRCs; this test notices when a change turns one coalesced copy
into several, moves traffic from one ingest path to another or stops counting something.  A change that alters a number on purpose
updates it here and says why."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FIELDS = ("memcpy_calls", "memcpy_bytes", "register_calls", "h2d_bytes", "blocks", "verified", "reg_hits", "reg_misses", "reg_rejected", "dma_jobs", "dma_bytes", "gds_bytes")

# case "tier/copy_group/call" -> FIELDS.  Tiers: arena = DMA out of pinned arena segments (2 MB register slices), files = registered
# mappings of the block files (registered inline), ring = pread into the pinned ring, framed = the worker's response stream received
# verbatim, ssd = disk-tier blocks through the GDS path.  Calls: whole file, a ranged read with partial first and last blocks, a vectored
# read with 37 boundary blocks (several staging rounds), a FUSE-shaped read, a shard of three, a small-file batch, a file with hole blocks.
# read_many goes through a reader of its own, so the per-reader device_stats fields stay 0 there.
# Within a group, pieces that follow on in the source (a pinned segment slice, a registered mapping, a super-slot that mirrors the
# destination) and in the destination share one copy.
EXPECTED = {
    "arena/cg1/whole": (43, 5249596, 0, 5247880, 41, 41, 0, 0, 0, 41, 5247880, 0),
    "arena/cg1/ranged": (23, 2622564, 0, 2621440, 21, 19, 0, 0, 0, 21, 2621440, 0),
    "arena/cg1/readv": (50, 5252868, 0, 5247880, 41, 41, 0, 0, 0, 41, 5247880, 0),
    "arena/cg1/fuse": (9, 671825, 0, 655377, 6, 4, 0, 0, 0, 6, 655377, 0),
    "arena/cg1/sharded": (16, 1710032, 0, 1708936, 14, 14, 0, 0, 0, 14, 1708936, 0),
    "arena/cg1/read_many": (21, 1795160, 0, 0, 0, 0, 0, 0, 0, 18, 1794048, 0),
    "arena/cg1/hole": (36, 4201020, 0, 4199304, 41, 33, 0, 0, 0, 33, 4199304, 0),
    "arena/cg4/whole": (13, 5249596, 0, 5247880, 41, 41, 0, 0, 0, 41, 5247880, 0),
    "arena/cg4/ranged": (8, 2622564, 0, 2621440, 21, 19, 0, 0, 0, 21, 2621440, 0),
    "arena/cg4/readv": (20, 5252340, 0, 5247880, 41, 41, 0, 0, 0, 41, 5247880, 0),
    "arena/cg4/fuse": (5, 671825, 0, 655377, 6, 4, 0, 0, 0, 6, 655377, 0),
    "arena/cg4/sharded": (16, 1710032, 0, 1708936, 14, 14, 0, 0, 0, 14, 1708936, 0),
    "arena/cg4/read_many": (8, 1795160, 0, 0, 0, 0, 0, 0, 0, 18, 1794048, 0),
    "arena/cg4/hole": (29, 4201020, 0, 4199304, 41, 33, 0, 0, 0, 9, 1053576, 0),
    "files/cg1/whole": (43, 5249596, 41, 5247880, 41, 41, 0, 41, 0, 0, 0, 0),
    "files/cg1/ranged": (23, 2622564, 21, 2621440, 21, 19, 0, 21, 0, 0, 0, 0),
    "files/cg1/readv": (50, 5252868, 41, 5247880, 41, 41, 0, 41, 0, 0, 0, 0),
    "files/cg1/fuse": (9, 671825, 6, 655377, 6, 4, 0, 6, 0, 0, 0, 0),
    "files/cg1/sharded": (16, 1710032, 14, 1708936, 14, 14, 0, 14, 0, 0, 0, 0),
    "files/cg1/read_many": (20, 1795160, 18, 0, 0, 0, 0, 0, 0, 0, 0, 0),
    "files/cg1/hole": (35, 4201020, 33, 4199304, 41, 33, 0, 33, 0, 0, 0, 0),
    "files/cg4/whole": (13, 5249596, 11, 5247880, 41, 41, 0, 11, 0, 0, 0, 0),
    "files/cg4/ranged": (8, 2622564, 6, 2621440, 21, 19, 0, 6, 0, 0, 0, 0),
    "files/cg4/readv": (18, 5252340, 11, 5247880, 41, 41, 0, 11, 0, 0, 0, 0),
    "files/cg4/fuse": (5, 671825, 2, 655377, 6, 4, 0, 2, 0, 0, 0, 0),
    "files/cg4/sharded": (6, 1710032, 4, 1708936, 14, 14, 0, 4, 0, 0, 0, 0),
    "files/cg4/read_many": (7, 1795160, 5, 0, 0, 0, 0, 0, 0, 0, 0, 0),
    "files/cg4/hole": (29, 4201020, 3, 4199304, 41, 33, 0, 3, 0, 0, 0, 0),
    "ring/cg1/whole": (43, 5249596, 0, 5247880, 41, 41, 0, 0, 0, 0, 0, 0),
    "ring/cg1/ranged": (23, 2622564, 0, 2621440, 21, 19, 0, 0, 0, 0, 0, 0),
    "ring/cg1/readv": (50, 5252868, 0, 5247880, 41, 41, 0, 0, 0, 0, 0, 0),
    "ring/cg1/fuse": (9, 671825, 0, 655377, 6, 4, 0, 0, 0, 0, 0, 0),
    "ring/cg1/sharded": (16, 1710032, 0, 1708936, 14, 14, 0, 0, 0, 0, 0, 0),
    "ring/cg1/read_many": (20, 1795160, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0),
    "ring/cg1/hole": (35, 4201020, 0, 4199304, 41, 33, 0, 0, 0, 0, 0, 0),
    "ring/cg4/whole": (13, 5249596, 0, 5247880, 41, 41, 0, 0, 0, 0, 0, 0),
    "ring/cg4/ranged": (8, 2622564, 0, 2621440, 21, 19, 0, 0, 0, 0, 0, 0),
    "ring/cg4/readv": (20, 5252340, 0, 5247880, 41, 41, 0, 0, 0, 0, 0, 0),
    "ring/cg4/fuse": (5, 671825, 0, 655377, 6, 4, 0, 0, 0, 0, 0, 0),
    "ring/cg4/sharded": (6, 1710032, 0, 1708936, 14, 14, 0, 0, 0, 0, 0, 0),
    "ring/cg4/read_many": (7, 1795160, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0),
    "ring/cg4/hole": (29, 4201020, 0, 4199304, 41, 33, 0, 0, 0, 0, 0, 0),
    "framed/cg1/whole": (54, 5253998, 0, 5249662, 41, 41, 0, 0, 0, 0, 0, 0),
    "framed/cg1/ranged": (29, 2690219, 0, 2687755, 21, 19, 0, 0, 0, 0, 0, 0),
    "framed/cg1/readv": (62, 5257270, 0, 5249662, 41, 41, 0, 0, 0, 0, 0, 0),
    "framed/cg1/fuse": (11, 736967, 0, 720139, 6, 4, 0, 0, 0, 0, 0, 0),
    "framed/cg1/sharded": (20, 1711518, 0, 1709530, 14, 14, 0, 0, 0, 0, 0, 0),
    "framed/cg1/read_many": (25, 1796948, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0),
    "framed/cg1/hole": (46, 4205006, 0, 4200734, 41, 33, 0, 0, 0, 0, 0, 0),
    "framed/cg4/whole": (24, 5375558, 0, 5371222, 41, 41, 0, 0, 0, 0, 0, 0),
    "framed/cg4/ranged": (14, 2816680, 0, 2814216, 21, 19, 0, 0, 0, 0, 0, 0),
    "framed/cg4/readv": (28, 5378302, 0, 5371222, 41, 41, 0, 0, 0, 0, 0, 0),
    "framed/cg4/fuse": (7, 754174, 0, 737346, 6, 4, 0, 0, 0, 0, 0, 0),
    "framed/cg4/sharded": (10, 1752038, 0, 1750050, 14, 14, 0, 0, 0, 0, 0, 0),
    "framed/cg4/read_many": (12, 2226544, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0),
    "framed/cg4/hole": (24, 5105158, 0, 5100886, 41, 33, 0, 0, 0, 0, 0, 0),
    "ssd/cg1/whole": (2, 1716, 0, 0, 41, 41, 0, 0, 0, 0, 0, 5247880),
    "ssd/cg1/ranged": (2, 1124, 0, 0, 21, 19, 0, 0, 0, 0, 0, 2621440),
    "ssd/cg1/readv": (9, 4988, 0, 0, 41, 41, 0, 0, 0, 0, 0, 5247880),
    "ssd/cg1/fuse": (3, 16448, 0, 0, 6, 4, 0, 0, 0, 0, 0, 655377),
    "ssd/cg1/sharded": (2, 1096, 0, 0, 14, 14, 0, 0, 0, 0, 0, 1708936),
    "ssd/cg1/read_many": (2, 1112, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0),
    "ssd/cg1/hole": (2, 1716, 0, 0, 41, 33, 0, 0, 0, 0, 0, 4199304),
    "ssd/cg4/whole": (2, 1716, 0, 0, 41, 41, 0, 0, 0, 0, 0, 5247880),
    "ssd/cg4/ranged": (2, 1124, 0, 0, 21, 19, 0, 0, 0, 0, 0, 2621440),
    "ssd/cg4/readv": (6, 4460, 0, 0, 41, 41, 0, 0, 0, 0, 0, 5247880),
    "ssd/cg4/fuse": (3, 16448, 0, 0, 6, 4, 0, 0, 0, 0, 0, 655377),
    "ssd/cg4/sharded": (2, 1096, 0, 0, 14, 14, 0, 0, 0, 0, 0, 1708936),
    "ssd/cg4/read_many": (2, 1112, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0),
    "ssd/cg4/hole": (26, 3147444, 0, 3145728, 41, 33, 0, 0, 0, 0, 0, 1053576),
}


def test_copy_shapes_of_every_ingest_path_are_pinned():
    sys.path.insert(0, os.path.join(ROOT, "tests", "mock_cuda"))
    try:
        import build as mock_build
    finally:
        sys.path.pop(0)
    env = dict(os.environ, CV_TEST_MOCK_CUDA_LIB=mock_build.build(), MOCK_CUDA_GDS="1")
    env.pop("MOCK_CUDA_ASYNC", None)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "mock_cuda", "copy_shapes.py")], cwd=ROOT, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert tuple(out["fields"]) == FIELDS
    got = {k: tuple(v) for k, v in out["cases"].items()}
    assert sorted(got) == sorted(EXPECTED)
    diff = {k: {f: (EXPECTED[k][i], got[k][i]) for i, f in enumerate(FIELDS) if EXPECTED[k][i] != got[k][i]} for k in EXPECTED if got[k] != EXPECTED[k]}
    assert not diff, "case -> field -> (pinned, got): %s" % json.dumps(diff, indent=1)
