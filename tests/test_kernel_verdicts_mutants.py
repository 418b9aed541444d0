"""The verdict tests (tests/test_zzz_kernel_verdicts_gpu.py) catch the bugs they are there for, and nothing else.

Each planted bug of tests/simt_emu/build.py's MUTATIONS below is built into the SIMT shim (the kernel source compiled for host cores), and
the verdict file runs against that library in a subprocess: the tests aimed at the bug must fail and every other test must pass; against
the library built from the unmodified source every test passes.  Without the verdict file, the `-m gpu` suite on the shim passes with
k2_ignores_header_len, k2_ignores_code, k2_compares_req_id_low_words or verify_marks_only_mismatches in; it catches
k2_rejects_16_mib_of_data only because one reader test happens to read with a 16 MB chunk, k2_ignores_total_len with one test, and the
two other verify bugs only through reader tests whose block layouts happen to put several mismatches in one warp or a skipped block
beside a mismatch.  Host memory only: nothing here touches a GPU."""
import re
from concurrent.futures import ThreadPoolExecutor

from test_launch_shapes_mutants import _outcomes
from test_simt_emu import _emu_build

FILES = ["tests/test_zzz_kernel_verdicts_gpu.py"]
FIELDS = r"::test_k2_flags_one_field_at_a_time\[%s-[01]\]"
# sizes with more than one entry in a warp: n = 1 cannot tell one count per warp from one per entry
WIDE = r"\[(31|32|33|255|256|257|1000003)\]"

# planted bug -> the tests aimed at it (a regular expression over test ids)
AIMED = {
    "k2_ignores_header_len": FIELDS % "header_len",
    "k2_ignores_code": FIELDS % "code",
    # data lengths set through total_len (every one disagrees with its descriptor) and total_len itself
    "k2_ignores_total_len": FIELDS % "(total_len|data_len)",
    # the high-word and sign-bit variants
    "k2_compares_req_id_low_words": FIELDS % "req_id",
    # a prefix that claims exactly 16 MiB, and a real 16 MiB frame
    "k2_rejects_16_mib_of_data": r"(%s|::test_k2_accepts_a_frame_of_exactly_16_mib\[)" % (FIELDS % "data_len"),
    "verify_counts_warps": r"::test_verify_crcs_\w+" + WIDE,
    "verify_ignores_the_skip_mask": r"::test_verify_crcs_masked_leaves_skipped_entries_out\[",
    # masks are guard-filled: every verify test that passes one
    "verify_marks_only_mismatches": r"::test_verify_crcs_\w+\[",
}


def test_each_planted_bug_fails_exactly_the_tests_aimed_at_it():
    b = _emu_build()
    libs = {"": b.build()}
    libs.update({m: b.build(mutate=m) for m in AIMED})
    with ThreadPoolExecutor(4) as pool:
        results = dict(zip(libs, pool.map(lambda lib: _outcomes(lib, FILES), libs.values())))
    clean = results.pop("")
    assert len(clean) >= 40 and all(v == "PASSED" for v in clean.values()), sorted((t, v) for t, v in clean.items() if v != "PASSED")
    for m, out in results.items():
        assert sorted(out) == sorted(clean), (m, "the file ran other tests than at the clean build")
        aimed = {t for t in out if re.search(AIMED[m], t)}
        assert aimed, (m, "no test is aimed at the bug")
        missed = sorted(t for t in aimed if out[t] not in ("FAILED", "CRASHED"))
        assert not missed, (m, "tests that should catch the bug passed", missed)
        broken = sorted(t for t in out if t not in aimed and out[t] not in ("PASSED", "SKIPPED"))
        assert not broken, (m, "tests not aimed at the bug failed", broken)
