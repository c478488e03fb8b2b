# Convenience targets over __graft_entry__.py / pytest / bench.py.
PY ?= python

.PHONY: build test test-gpu bench bench-ref stress clean

build:            ## libbsgpu.so (nvcc, sm_90a) + the CPU oracle; no GPU needed
	$(PY) __graft_entry__.py

test: build       ## CPU suite: oracle vs the reference's fixtures, ABI, layout models, gloo sharding
	$(PY) -m pytest tests -x -q -m "not gpu"

test-gpu: build   ## parity tests through the C ABI (needs an H100)
	$(PY) -m pytest tests -x -q -m gpu

bench: build      ## headline benchmark, one GPU
	$(PY) bench.py

bench-ref: build  ## the CPU arm (oracle port of bed_pMatVec4 on the host cores)
	$(PY) bench.py --impl reference

stress: build     ## randomised GPU-vs-oracle sweep
	$(PY) tools/stress.py --cases 150

clean:
	rm -f bigsnpr_b200/libbsgpu.so
	rm -rf oracle/_build
