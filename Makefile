# Convenience targets over __graft_entry__.build(), pytest and bench.py.
PY ?= python

build:            ## libcurvine_b200.so (nvcc, sm_90a; no GPU needed) + the oracle's C restatement
	$(PY) __graft_entry__.py

test:             ## CPU suite (oracle, host side, stand-in runtime, kernel source on the SIMT shim)
	$(PY) -m pytest tests -x -q -m "not gpu"

test-gpu:         ## parity suite on an H100
	$(PY) -m pytest tests -x -q -m gpu

sanitize:         ## host ASan/UBSan + TSan, GPU reader on the stand-in runtime (incl. stream order), kernel source on the shim
	bash tools/sanitize_host.sh
	bash tools/tsan_host.sh
	bash tools/sanitize_ingest.sh
	bash tools/sanitize_kernels.sh full
	$(PY) -m curvine_b200.build

bench:            ## the BASELINE.json metric on one GPU, and the reference's CPU path beside it
	$(PY) bench.py --gpus 1
	$(PY) bench.py --impl reference --gpus 1

example:          ## the plain-C host of INTEGRATION.md
	gcc -std=c99 -Wall -Wextra -pedantic -I include examples/c_host.c -o examples/c_host -L curvine_b200 -l:libcurvine_b200.so -Wl,-rpath,$(CURDIR)/curvine_b200

.PHONY: build test test-gpu sanitize bench example
