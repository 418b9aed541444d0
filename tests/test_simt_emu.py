"""The product's KERNEL SOURCE on a machine without a GPU.

tests/simt_emu compiles curvine_b200/csrc/kernels.cu -- the file nvcc compiles for sm_90a, unmodified apart from a mechanical
rewrite of the launch syntax and of the inline PTX -- for host cores on a SIMT shim: a fiber per CUDA thread, blocks spread over
host threads, __syncthreads / __syncwarp / *_sync warp intrinsics completing exactly when every live participant has arrived.
The whole `-m gpu` suite (kernel parity against the oracle, the reader through the C ABI, arena, GDS fallback, faults, the
two-device gather) then runs in a subprocess against that library -- with the runtime stand-in's streams running ASYNCHRONOUSLY
(tests/mock_cuda/mock_cuda.cc: a thread per stream, random pauses, ordering only through events), so the pipeline's stream
dependencies are exercised too.  This checks the kernels' ALGORITHM (index math, shuffle
patterns, the GF(2) folds, barrier placement) on every CPU run; what it cannot check is what only the hardware decides (memory
model races between unsynchronised threads, the compiled SASS, speed) -- the H100 run of the same tests covers that.
Test infrastructure: nothing under curvine_b200/ can load this library."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run_suite_retrying_flakes(cmd, env, timeout):
    """Runs a pytest subprocess.  ~140 integration tests with worker processes, sockets and timeouts run 6-way parallel on a shared machine: a test
    that fails is run once more ON ITS OWN; a second failure fails this test, a pass is reported as a warning naming the flaky test (a flake of
    this kind exposed the connection-pool bug fixed in round 2, so it is worth reading)."""
    import warnings
    r = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout)
    if r.returncode == 0:
        return r.stdout
    failed = sorted(set(re.findall(r"^(?:FAILED|ERROR) (\S+)", r.stdout, re.M)))
    first_tail = "\n".join(r.stdout.splitlines()[-30:])
    assert failed and len(failed) <= 3, first_tail  # a crash, a collection error or a broad failure is not a flake
    ids = [os.path.join(ROOT, f.split("::")[0]) + "::" + "::".join(f.split("::")[1:]) for f in failed]
    again = subprocess.run([sys.executable, "-m", "pytest"] + ids + ["-m", "gpu", "-q", "-p", "no:cacheprovider"], cwd=ROOT, env=env, stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, text=True, timeout=timeout)
    assert again.returncode == 0, first_tail + "\n---- second run of the failed tests ----\n" + "\n".join(again.stdout.splitlines()[-30:])
    warnings.warn("flaky under load, passed when run again on their own: %s\n%s" % (", ".join(failed), first_tail))
    return re.sub(r"(\d+) failed, (\d+) passed", lambda m: "%d passed" % (int(m.group(1)) + int(m.group(2))), r.stdout)


def _emu_build():
    # tests/mock_cuda/build.py is a module called `build` too: load this one by path
    import importlib.util
    spec = importlib.util.spec_from_file_location("simt_emu_build", os.path.join(ROOT, "tests", "simt_emu", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_shim_known_answers_and_deadlock_report():
    exe = _emu_build().build_selftest()
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=120)
    assert r.returncode == 0 and "selftest ok" in r.stdout, r.stdout
    for name in ("scan", "early_exit", "smem_ptx", "launch_errors"):
        assert name + " ok" in r.stdout, r.stdout
    # a barrier part of the block never reaches is reported, not spun on
    r = subprocess.run([exe, "deadlock"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=60)
    assert r.returncode != 0 and "deadlock in block 0" in r.stdout and "not reached" not in r.stdout, r.stdout


def test_rewrite_refuses_unknown_forms_and_covers_the_kernel_file():
    b = _emu_build()
    ok = b.rewrite('__global__ void k(int* p) { asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(a), "r"(b), "r"(c), "r"(d) : "memory"); }\n'
                   'void f() { k<<<1, 32, 0, st>>>(p); }')
    assert "cv_emu::ptx_st_v4((p), (a), (b), (c), (d))" in ok and "cv_emu::cfg(1, 32, 0, st)(k, p)" in ok and "<<<" not in ok
    with pytest.raises(ValueError, match="does not know"):
        b.rewrite('void f() { asm volatile("tcgen05.mma.cta_group::1.kind::f16 [%0], %1, %2, %3, p;" ::"r"(d), "l"(a), "l"(b), "r"(i)); }')
    with pytest.raises(ValueError, match="launch configuration"):
        b.rewrite("void f() { k<<<1, 32>>>(p); }")
    # every asm statement and launch of the product's kernel file is understood, and nothing CUDA-only is left for g++
    out = b.rewrite(open(os.path.join(ROOT, "curvine_b200", "csrc", "kernels.cu")).read())
    assert "<<<" not in out and not re.search(r"\basm\b", out) and "extern __shared__" not in out
    assert out.count("cv_emu::cfg(") == 22 and out.count("\n") == open(os.path.join(ROOT, "curvine_b200", "csrc", "kernels.cu")).read().count("\n")


def test_gpu_suite_with_the_kernel_source_on_the_simt_shim():
    lib = _emu_build().build()
    # MOCK_CUDA_ASYNC: the runtime stand-in runs every created stream as a FIFO of its own with random pauses, ordered only by events --
    # a dependency the pipeline forgot between its copy / verify / caller streams shows up as wrong bytes (tools/sanitize_ingest.sh plants one)
    env = dict(os.environ, CV_TEST_MOCK_CUDA_LIB=lib, CV_SIMT_EMU_THREADS="3", MOCK_CUDA_ASYNC="1", MOCK_CUDA_JITTER_US="500")
    out = _run_suite_retrying_flakes([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests"), "-m", "gpu", "-q", "-p", "no:cacheprovider", "-n", "6"], env, 2400)
    tail = "\n".join(out.splitlines()[-30:])
    m = re.search(r"(\d+) passed", out)
    assert m and int(m.group(1)) >= 142, tail


def test_sanitizer_builds_of_the_shim_report_planted_bugs_and_nothing_else():
    """tools/sanitize_kernels.sh runs the kernel suites on the shim under ASan+UBSan and under TSan (as a race check between CUDA
    threads).  Here: the shim's known-answer program in both builds -- a planted out-of-bounds store, an out-of-bounds granule load
    and planted races (missing barrier inside a block, plain add from two blocks) ARE reported, their correct twins are not."""
    b = _emu_build()
    env = dict(os.environ, ASAN_OPTIONS="detect_stack_use_after_return=0:detect_leaks=0", TSAN_OPTIONS="halt_on_error=0 history_size=4", CV_SIMT_EMU_THREADS="2")

    def run(exe, *args, wrap=()):
        return subprocess.run(list(wrap) + [exe] + list(args), env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300).stdout

    exe = b.build_selftest("address")
    assert "selftest ok" in run(exe)
    assert "heap-buffer-overflow" in run(exe, "oob", "1") and "heap-buffer-overflow" in run(exe, "oob", "2")
    out = run(exe, "oob", "3")  # reading the rest of the last 16-byte granule of a buffer is the kernels' documented behaviour
    assert "AddressSanitizer" not in out and "oob kernel done" in out
    exe = b.build_selftest("thread")
    wrap = ("setarch", os.uname().machine, "-R")  # TSan wants a fixed address-space layout on this kernel
    assert "selftest ok" in run(exe, wrap=wrap) and "data race" not in run(exe, wrap=wrap)
    for k, racy in ((0, True), (1, False), (2, False), (3, True), (4, False), (5, True), (6, False)):
        out = run(exe, "race", str(k), wrap=wrap)
        assert ("ThreadSanitizer: data race" in out) == racy and "race kernel done" in out, (k, out[-2000:])
