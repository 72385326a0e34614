# Convenience targets; the driver uses __graft_entry__.build(), pytest and bench.py directly.
PY ?= python

build:            ## nvcc -gencode arch=compute_90a,code=sm_90a -> libcdprobe.so, g++ -> cdprobe-daemon, gcc -> oracle
	$(PY) -c "import __graft_entry__ as g; g.build()"

test: build       ## CPU suite (no GPU needed)
	$(PY) -m pytest tests -x -q -m "not gpu"

test-gpu: build   ## parity suite on an H100
	$(PY) -m pytest tests -x -q -m gpu

bench: build      ## one JSON line (N = 1); N > 1: python -m torch.distributed.run --nproc-per-node N bench.py --gpus N
	$(PY) bench.py --gpus 1

golden:           ## regenerate tests/golden/golden.json from the pure-Python statement
	$(PY) tests/golden/make_golden.py

clean:
	rm -f k8s-dra-driver-gpu_b200/libcdprobe.so k8s-dra-driver-gpu_b200/cdprobe-daemon
	$(MAKE) -C oracle clean

.PHONY: build test test-gpu bench golden clean
