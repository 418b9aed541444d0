#!/bin/bash
# Host-side C++ (worker threads, client connection pool, parallel readers) under ThreadSanitizer.
# Same scheme as sanitize_host.sh: sanitized copy of the library in /tmp, swapped in for the CPU host tests, restored afterwards.
set -e
ROOT="$(cd "$(dirname "$0")/.." && pwd)"
W=/tmp/cv_tsan; mkdir -p $W; cd $W
for f in $ROOT/curvine_b200/csrc/kernels.cu $ROOT/curvine_b200/csrc/host/*.cu $ROOT/curvine_b200/csrc/host/*.cc; do
  x=cu; case $f in *.cc) x=c++;; esac
  nvcc -gencode arch=compute_90a,code=sm_90a -O1 -g -std=c++17 \
    -Xcompiler -fPIC,-pthread,-msse4.2,-fsanitize=thread,-fno-omit-frame-pointer -cudart static \
    -I $ROOT/include -I $ROOT/curvine_b200/csrc -x $x -c $f -o $(basename $f).o &
done; wait
nvcc -gencode arch=compute_90a,code=sm_90a -shared -cudart static -Xcompiler -fsanitize=thread -o tsan.so *.o -lpthread -ldl -lrt
cp $ROOT/curvine_b200/libcurvine_b200.so orig.so; cp tsan.so $ROOT/curvine_b200/libcurvine_b200.so
trap "cp $W/orig.so $ROOT/curvine_b200/libcurvine_b200.so" EXIT
cd $ROOT
LD_PRELOAD="$(gcc -print-file-name=libtsan.so)" TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0 history_size=4 ${TSAN_EXTRA}" \
  setarch "$(uname -m)" -R python -m pytest tests/test_host.py tests/test_arena.py tests/test_hostile_peers.py -q -p no:cacheprovider -s -x ${TSAN_TESTS} 2>&1 | tee $W/report.txt | tail -5
echo "tsan findings: $(grep -c 'WARNING: ThreadSanitizer' $W/report.txt)"
