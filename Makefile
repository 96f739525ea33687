# Build / test entry points (reference: Makefile:40-90 + .github/workflows/main.yml). The real build logic lives in
# distributed_llama_b200/_build.py (g++ for the host library and native front ends, nvcc -gencode arch=compute_90a,code=sm_90a
# for the CUDA library); these targets only name the common invocations.
PY ?= python

.PHONY: all build host cuda native test test-gpu bench smoke sanitize clean

all: build

build:            ## host library, CUDA library, dllama-native, dllama-api-native
	$(PY) -m distributed_llama_b200._build

native: build

test:             ## CPU tests (formats, tokenizer, converters, apps, native API server, reference-binary parity)
	$(PY) -m pytest tests -q -m "not gpu"

test-gpu:         ## needs an H100
	$(PY) -m pytest tests -q -m gpu

bench:
	$(PY) bench.py --gpus 1 --steps 64 --warmup 8

smoke:
	$(PY) -c "import __graft_entry__ as g; g.build(); g.smoke()"

sanitize:         ## compute-sanitizer memcheck over every kernel family (needs an H100)
	bash tools/sanitize.sh memcheck

clean:
	rm -rf build distributed_llama_b200/*.so distributed_llama_b200/*.hash distributed_llama_b200/dllama-native distributed_llama_b200/dllama-api-native
