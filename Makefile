# Convenience targets (__graft_entry__.build() runs the same commands).
.PHONY: all lib oracle ref cpp test clean
all: lib oracle cpp

lib:            ## libsrtb_b200.so (nvcc, sm_90a only)
	simple-radio-telescope-backend_b200/csrc/build.sh

oracle:         ## CPU oracle (test infrastructure)
	$(MAKE) -C oracle libsrtb_oracle.so

ref:            ## the reference's own headers through the host SYCL shim (needs /root/reference)
	$(MAKE) -C oracle ref

cpp: lib        ## C++ pipe framework tests + pipeline_main (the reference's main.cpp wiring on the re-hosted pipes)
	$(MAKE) -C tests/cpp all

test:           ## CPU-only suite; add `-m gpu` on an H100
	python -m pytest tests -q -m "not gpu"

clean:
	$(MAKE) -C tests/cpp clean
	rm -f simple-radio-telescope-backend_b200/csrc/*.so oracle/*.so
