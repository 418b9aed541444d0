"""The loads of the official writer's checkpoints (tests/test_zzz_checkpoint_interop_gpu.py) catch bugs the older files miss.

Each planted bug of tests/simt_emu/build.py's MUTATIONS below is built into the SIMT shim (the kernel and host sources compiled for host
cores), and the new file runs against that library in a subprocess.  The tests aimed at the bug must fail and every other test must
pass; the pre-existing `-m gpu` suite passes with either bug in.  Both bugs live where only the new file's loads reach: converting rows
split by a block edge for a dtype pair the older loads never split, and block lengths that are not a multiple of 16 bytes (every older
file uses 64 KiB or 4 MiB blocks).  Two bugs in the scaled path were tried first and not kept, because the older suite already fails
with them in: a scaled span's view position that keeps only its offset inside its row, and a scale walk that keeps the old scale when
a chunk steps from a view row's end into the next row of tiles.  Host memory only: nothing here touches a GPU."""
import re
from concurrent.futures import ThreadPoolExecutor

from test_launch_shapes_mutants import _outcomes
from test_simt_emu import _emu_build

FILES = ["tests/test_zzz_checkpoint_interop_gpu.py"]

# planted bug -> the tests aimed at it (a regular expression over test ids)
AIMED = {
    # the rest of an F16 -> F32 row that crosses a block edge lands at its source offset: the float32 loads at odd block sizes
    "cast_row_rest_offset_in_source_bytes": r"::test_official_checkpoints_load_as_the_numpy_reference\[",
    # staging slots spaced by the block length rounded down to 16 bytes overlap at 12292-byte blocks: loads that stage 2+ blocks
    "readv_stage_slots_rounded_down_to_16": r"::test_official_checkpoints_load_as_the_numpy_reference\[",
}


def test_each_planted_bug_fails_exactly_the_tests_aimed_at_it():
    b = _emu_build()
    libs = {m: b.build(mutate=m) for m in AIMED}
    with ThreadPoolExecutor(len(libs)) as pool:
        results = dict(zip(libs, pool.map(lambda lib: _outcomes(lib, FILES), libs.values())))
    for m, out in results.items():
        assert len(out) >= 10, (m, out)
        aimed = {t for t in out if re.search(AIMED[m], t)}
        assert aimed, (m, "no test is aimed at the bug")
        missed = sorted(t for t in aimed if out[t] not in ("FAILED", "CRASHED"))
        assert not missed, (m, "tests that should catch the bug passed", missed)
        broken = sorted(t for t in out if t not in aimed and out[t] not in ("PASSED", "SKIPPED"))
        assert not broken, (m, "tests not aimed at the bug failed", broken)
