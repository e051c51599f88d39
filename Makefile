# Thin wrapper: the real build lives in faabric_b200/build.py (nvcc sm_90a + g++)
PY ?= python

.PHONY: all build test test-gpu cpp-test bench clean
all: build

build:
	$(PY) -m faabric_b200.build

test: build
	$(PY) -m pytest tests -x -q -m "not gpu"

test-gpu: build
	$(PY) -m pytest tests -x -q -m gpu

cpp-test: build
	build/bin/faabric_tests

bench: build
	$(PY) bench.py

clean:
	rm -rf build faabric_b200/lib
