"""The launch-shape tests (tests/test_zzz_launch_shapes_gpu.py) catch the bugs they are there for.

Each planted bug of tests/simt_emu/build.py's MUTATIONS below is built into the SIMT shim (the kernel source compiled for host
cores), and the launch-shape file runs against that library in a subprocess.  The tests aimed at the bug must fail and every other
test must pass; the pre-existing kernel suites pass with both bugs in, which is why the launch-shape file exists.  Host memory only:
nothing here touches a GPU.  A test the subprocess dies in counts as failed, and the rest of the file runs again without it."""
import os
import re
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

from test_simt_emu import _emu_build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILE = "tests/test_zzz_launch_shapes_gpu.py"

# planted bug -> the tests aimed at it (a regular expression over test ids)
AIMED = {
    # the shifted walk keeps only 1023 rows of 512 bytes: units of 2^19 and 2^20 bytes from a source at another 16-byte phase
    "shifted_walk_drops_rows_past_1023": r"::test_(k2_k4_frames_around|k3_gather_pages|gather_strided_rows|deinterleave_and_p2p)\w*\[s(19|20)\b",
    # K5's scale walk divides in 32 bits: every test with a view position or width past 2^32
    "scale_walk_divides_in_32_bits": r"::test_(k5_scaled_views_past_2_32|scaled_reads_with_view_positions_past_2_32|the_last_scale_of_a_wide_view)\w*\[",
}


def _outcomes(lib):
    """{test id: PASSED / FAILED / ERROR / SKIPPED / CRASHED} of the launch-shape file against `lib`"""
    env = dict(os.environ, CV_TEST_MOCK_CUDA_LIB=lib, CV_SIMT_EMU_THREADS="4")
    for k in ("MOCK_CUDA_ASYNC", "MOCK_CUDA_JITTER_US", "CV_SIMT_EMU_SMS"):
        env.pop(k, None)
    done = {}
    while True:
        cmd = [sys.executable, "-m", "pytest", FILE, "-m", "gpu", "-v", "-p", "no:cacheprovider"]
        cmd += ["--deselect=" + t for t in done]
        r = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
        for t, what in re.findall(r"^(\S+::\S+) (PASSED|FAILED|ERROR|SKIPPED)\b", r.stdout, re.M):
            done[t] = what
        if r.returncode in (0, 1):
            return done
        # the process died: the last test it started has no outcome on its line
        started = [line.split()[0] for line in r.stdout.splitlines() if re.match(r"\S+::\S+", line)]
        assert started and started[-1] not in done, "\n".join(r.stdout.splitlines()[-30:])
        done[started[-1]] = "CRASHED"


def test_each_planted_bug_fails_exactly_the_tests_aimed_at_it():
    b = _emu_build()
    libs = {m: b.build(mutate=m) for m in AIMED}
    with ThreadPoolExecutor(len(libs)) as pool:
        results = dict(zip(libs, pool.map(_outcomes, libs.values())))
    for m, out in results.items():
        assert len(out) > 80, (m, out)
        aimed = {t for t in out if re.search(AIMED[m], t)}
        assert len(aimed) >= 6, (m, sorted(aimed))
        missed = sorted(t for t in aimed if out[t] not in ("FAILED", "CRASHED"))
        assert not missed, (m, "tests that should catch the bug passed", missed)
        broken = sorted(t for t in out if t not in aimed and out[t] not in ("PASSED", "SKIPPED"))
        assert not broken, (m, "tests not aimed at the bug failed", broken)
