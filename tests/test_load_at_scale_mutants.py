"""The full-size load and K5 depth tests catch the bugs they are there for.

Each planted bug of tests/simt_emu/build.py's MUTATIONS below is built into the SIMT shim (the kernel and host sources compiled for
host cores), and the three files of those tests run against that library in a subprocess.  The tests aimed at the bug must fail and
every other test must pass; the pre-existing `-m gpu` suite passes with either bug in.  Host memory only: nothing here touches a GPU.
A test the subprocess dies in counts as failed, and the rest of the files run again without it."""
import re
from concurrent.futures import ThreadPoolExecutor

from test_launch_shapes_mutants import _outcomes
from test_simt_emu import _emu_build

FILES = ["tests/test_zzz_cast_exhaustive_gpu.py", "tests/test_zzz_cast_at_depth_gpu.py", "tests/test_zzz_readv_at_scale_gpu.py"]

# planted bug -> the tests aimed at it (a regular expression over test ids)
AIMED = {
    # K5's segment search resolves at most 64 segments: the depth tables, whose grid strides skip thousands of segments, and the
    # converting dim-1 slices of the full-size loads, whose rounds hold one segment per row that crosses a block
    "cast_segment_search_spans_64_segments": r"(test_zzz_cast_at_depth_gpu\.py::test_(plain|scaled)_instance_at_full_grid_depth\[|"
                                             r"::test_tensor_parallel_slices\[\w+-1-bfloat16\]|::test_fp8_dequantized_loads\[arena-True\])",
    # readv_device keeps a span's offset inside its range in 32 bits: the rows 4 GiB past their range's start
    "readv_row_offset_32_bits": r"::test_destinations_more_than_4_gib_apart$",
}


def test_each_planted_bug_fails_exactly_the_tests_aimed_at_it():
    b = _emu_build()
    libs = {m: b.build(mutate=m) for m in AIMED}
    with ThreadPoolExecutor(len(libs)) as pool:
        results = dict(zip(libs, pool.map(lambda lib: _outcomes(lib, FILES), libs.values())))
    for m, out in results.items():
        assert len(out) > 60, (m, out)
        aimed = {t for t in out if re.search(AIMED[m], t)}
        assert aimed, (m, "no test is aimed at the bug")
        missed = sorted(t for t in aimed if out[t] not in ("FAILED", "CRASHED"))
        assert not missed, (m, "tests that should catch the bug passed", missed)
        broken = sorted(t for t in out if t not in aimed and out[t] not in ("PASSED", "SKIPPED"))
        assert not broken, (m, "tests not aimed at the bug failed", broken)
