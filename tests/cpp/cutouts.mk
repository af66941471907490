# test_cutouts: CPU-only tests of the candidate cut-outs' host pieces (make -C tests/cpp -f cutouts.mk). Needs
# libsrtb_b200.so (built first) for its host symbols, and libcudart; no GPU.
CXX := /usr/bin/g++
ROOT := $(abspath ../..)
CUDA ?= /usr/local/cuda
LIBDIR := $(ROOT)/simple-radio-telescope-backend_b200/csrc
CXXFLAGS := -std=c++20 -O2 -Wall -pthread -I$(ROOT)/include

all: test_cutouts

test_cutouts: test_cutouts.cpp $(wildcard $(ROOT)/include/srtb/*.hpp $(ROOT)/include/srtb/pipeline/*.hpp $(ROOT)/include/srtb/io/*.hpp $(ROOT)/include/*.h) $(wildcard $(LIBDIR)/libsrtb_b200.so)
	@if [ -f $(LIBDIR)/libsrtb_b200.so ]; then \
	  $(CXX) $(CXXFLAGS) -I$(CUDA)/include -o $@ $< -L$(LIBDIR) -lsrtb_b200 -L$(CUDA)/lib64 -lcudart \
	    -Wl,-rpath,'$$ORIGIN/../../simple-radio-telescope-backend_b200/csrc' -Wl,-rpath,$(CUDA)/lib64; \
	else echo "libsrtb_b200.so missing: skipping test_cutouts"; fi

clean:
	rm -f test_cutouts
.PHONY: all clean
