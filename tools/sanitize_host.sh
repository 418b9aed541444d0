#!/bin/bash
# Host-side C++ under AddressSanitizer + UBSan (SURVEY.md §5: the reference has no sanitizer runs; this is our equivalent).
# Builds a sanitized copy of the library into /tmp, swaps it in for the CPU test suite, restores the real one.
set -e
ROOT="$(cd "$(dirname "$0")/.." && pwd)"
W=/tmp/cv_asan; mkdir -p $W; cd $W
for f in $ROOT/curvine_b200/csrc/kernels.cu $ROOT/curvine_b200/csrc/host/*.cu $ROOT/curvine_b200/csrc/host/*.cc; do
  x=cu; case $f in *.cc) x=c++;; esac
  nvcc -gencode arch=compute_90a,code=sm_90a -O1 -g -std=c++17 \
    -Xcompiler -fPIC,-pthread,-msse4.2,-fsanitize=address,-fsanitize=undefined,-fno-omit-frame-pointer -cudart static \
    -I $ROOT/include -I $ROOT/curvine_b200/csrc -x $x -c $f -o $(basename $f).o &
done; wait
nvcc -gencode arch=compute_90a,code=sm_90a -shared -cudart static -Xcompiler -fsanitize=address,-fsanitize=undefined -o asan.so *.o -lpthread -ldl -lrt
cp $ROOT/curvine_b200/libcurvine_b200.so orig.so; cp asan.so $ROOT/curvine_b200/libcurvine_b200.so
trap "cp $W/orig.so $ROOT/curvine_b200/libcurvine_b200.so" EXIT
cd $ROOT
LD_PRELOAD="$(gcc -print-file-name=libasan.so) $(gcc -print-file-name=libubsan.so)" ASAN_OPTIONS=detect_leaks=0:halt_on_error=0 \
  UBSAN_OPTIONS=print_stacktrace=1 python -m pytest tests/test_host.py tests/test_multi_cpu.py tests/test_arena.py tests/test_wire_pin.py tests/test_hostile_peers.py tests/test_curvinefs_compat.py -q -p no:cacheprovider -s 2>&1 | tee $W/report.txt | tail -5
echo "sanitizer findings: $(grep -ciE 'runtime error|AddressSanitizer' $W/report.txt)"
