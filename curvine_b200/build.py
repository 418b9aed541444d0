"""In-tree build of libcurvine_b200.so (CUDA kernels for sm_90a + C++ host library, one C-ABI .so).

nvcc cross-compiles without a GPU.  The built .so is git-ignored and lives in the source tree; nothing is
JIT-compiled at import time.
"""
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")
LIB = os.path.join(HERE, "libcurvine_b200.so")
STAMP = os.path.join(HERE, ".build_stamp")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC,-O3,-Wall,-pthread,-msse4.2", "-cudart", "static"]


def _nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def sources():
    out = []
    for root, _, files in os.walk(CSRC):
        for f in sorted(files):
            if f.endswith((".cu", ".cc")):
                out.append(os.path.join(root, f))
    return sorted(out)


def _digest():
    h = hashlib.sha256()
    for root in (CSRC, INCLUDE):
        for r, _, files in os.walk(root):
            for f in sorted(files):
                if f.endswith((".cu", ".cc", ".h", ".cuh")):
                    p = os.path.join(r, f)
                    h.update(p.encode())
                    h.update(open(p, "rb").read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP) and open(STAMP).read() == dig:
        return LIB
    objs = []
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    procs = []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src) + ".o")
        objs.append(obj)
        cmd = [_nvcc()] + NVCC_FLAGS + ["-I", INCLUDE, "-I", CSRC, "-x", "cu" if src.endswith(".cu") else "c++",
                                         "-c", src, "-o", obj]
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, out.decode()))
        if verbose and out:
            print(out.decode(), file=sys.stderr)
    cmd = [_nvcc()] + NVCC_FLAGS + ["-shared", "-o", LIB] + objs + ["-lpthread", "-ldl", "-lrt"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode:
        raise RuntimeError("link failed:\n" + r.stdout.decode())
    open(STAMP, "w").write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
