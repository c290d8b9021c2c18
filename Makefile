# Convenience targets (everything is plain python underneath).
PY ?= python

.PHONY: build test test-gpu bench smoke sass-check reference clean

build:            ## nvcc -gencode arch=compute_90a,code=sm_90a -> swiftllm_b200/libswiftllm_b200.so
	$(PY) -m swiftllm_b200.build

test: build       ## CPU suite: oracle vs golden vectors, host logic, C-ABI surface, gloo TP, dry runs, mirrors
	$(PY) -m pytest tests -q -m "not gpu"

test-gpu: build   ## parity through the C ABI on a B200 (multi-GPU cases skip themselves when the box has fewer devices)
	$(PY) -m pytest tests -q -m gpu

bench: build      ## one JSON line: decode tokens/s of BASELINE.json configs[1] on one B200
	$(PY) bench.py

smoke: build
	$(PY) -c "import __graft_entry__ as g; g.smoke()"

sass-check: build ## validated kernels still compile to their validated instruction streams
	$(PY) -m pytest tests/test_cabi.py -q -k validated

reference:        ## the unmodified reference under baseline/_ref (for scripts/ref_triton_bench.py / the reference_triton block of bench.py)
	bash scripts/install_reference.sh

clean:
	rm -rf swiftllm_b200/csrc/build swiftllm_b200/libswiftllm_b200.so
