"""The GPU ingest pipeline's HOST logic on a machine without a GPU.

tests/test_gpu_reader.py is the parity suite of the reader through the C ABI (`-m gpu`, run on an H100 against the real
library).  Here the same tests run in a subprocess against tests/mock_cuda's library: the product's C++ host side
(csrc/host/*: job planning, pinned ring, copy groups, registrar, fetch threads, verify batching, result harvesting, the
worker, the writer, the HBM tier) compiled against a host-memory stand-in for the CUDA runtime, with plain-loop CPU stand-ins
for the cvk_* launchers instead of csrc/kernels.cu.  That checks the pipeline's bookkeeping (what lands where, which CRC is
compared with which manifest entry, slot reuse, cache revalidation, error paths) on every CPU run; it says nothing about the
kernels (tests/test_simt_emu.py runs the same suites against the kernel SOURCE on a SIMT shim; the H100 run checks the compiled code).  The mock is test infrastructure: nothing under curvine_b200/ can load it."""
import os
import re
import subprocess
import sys

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


def test_gpu_reader_suite_against_the_mock_runtime_and_its_launcher_stand_ins():
    sys.path.insert(0, os.path.join(ROOT, "tests", "mock_cuda"))
    try:
        import build as mock_build
    finally:
        sys.path.pop(0)
    lib = mock_build.build()
    env = dict(os.environ, CV_TEST_MOCK_CUDA_LIB=lib)
    out = _run_suite_retrying_flakes([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_reader.py"), os.path.join(ROOT, "tests", "test_zz_gpu_reader_faults.py"),
                                      os.path.join(ROOT, "tests", "test_arena_gpu.py"), os.path.join(ROOT, "tests", "test_gds_gpu.py"), "-m", "gpu", "-q", "-p", "no:cacheprovider", "-n", "6"], env, 1500)
    tail = "\n".join(out.splitlines()[-25:])
    m = re.search(r"(\d+) passed", out)
    assert m and int(m.group(1)) >= 60, tail


def test_device_reader_on_the_mock_runtime_releases_every_device_and_pinned_allocation_and_registration():
    """tests/mock_cuda/leak_check.py: mixed workload over four pipeline configurations incl. failed and abandoned reads and a device
    write; after every cv_fs_close the mock runtime must hold no device allocation, no pinned allocation and no registered range."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "mock_cuda"))
    try:
        import build as mock_build
    finally:
        sys.path.pop(0)
    env = dict(os.environ, CV_TEST_MOCK_CUDA_LIB=mock_build.build())
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "mock_cuda", "leak_check.py")], cwd=ROOT, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0 and "leak check ok" in r.stdout, r.stdout[-3000:]
