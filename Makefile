# Convenience targets (the reference ships a Makefile only for its C++ index helpers; here everything native is built in-tree).
PY ?= python

.PHONY: build helpers test test-gpu smoke bench bench-ref clean

build:            ## nvcc -gencode arch=compute_90a,code=sm_90a -> relora_b200/_C.so ; g++ -> relora_b200/_data_helpers.so
	$(PY) -c "import __graft_entry__ as g; g.build()"

helpers:          ## only the C++17 / pybind11 dataset index builders
	$(PY) -m relora_b200.data.neox.helpers_build

test:             ## CPU / gloo suite
	$(PY) -m pytest tests -x -q -m "not gpu"

test-gpu:         ## kernel numerics + fused executor (needs an H100)
	$(PY) -m pytest tests -x -q -m gpu

smoke:
	$(PY) -c "import __graft_entry__ as g; g.smoke()"

bench:            ## headline metric, one JSON line
	$(PY) bench.py --gpus 1

bench-ref:        ## the unmodified reference from baseline/_ref
	$(PY) bench.py --impl reference --gpus 1

clean:
	rm -rf relora_b200/csrc/_build relora_b200/_C.so relora_b200/_data_helpers.so
