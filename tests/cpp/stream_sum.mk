# test_stream_sum: CPU-only tests of the total-intensity detector's host pieces (make -C tests/cpp -f stream_sum.mk).
# Links libcudart only; the test stands in for the device calls a cuda_queue makes, so it needs no GPU.
CXX := /usr/bin/g++
ROOT := $(abspath ../..)
CUDA ?= /usr/local/cuda
CXXFLAGS := -std=c++20 -O2 -Wall -pthread -I$(ROOT)/include

all: test_stream_sum

test_stream_sum: test_stream_sum.cpp $(wildcard $(ROOT)/include/srtb/*.hpp $(ROOT)/include/srtb/pipeline/*.hpp $(ROOT)/include/srtb/io/*.hpp $(ROOT)/include/*.h)
	$(CXX) $(CXXFLAGS) -I$(CUDA)/include -o $@ $< -L$(CUDA)/lib64 -lcudart -Wl,-rpath,$(CUDA)/lib64

clean:
	rm -f test_stream_sum
.PHONY: all clean
