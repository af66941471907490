// src/correlator.cpp — `srtb_b200_correlator`, the basic baseband correlator (the reference's
// userspace/src/correlator.cpp): reads two recordings of unsigned 8-bit samples (two polarisations or two antennas),
// forms their cross spectrum and writes the magnitude of the cross-correlation, complex_count = min(size) / 2 raw
// float32 values, as the reference writes them. The device work is one srtb_b200_correlate call.
//
//   srtb_b200_correlator [--input_file_1 pol_1.bin] [--input_file_2 pol_2.bin] [--output_file /dev/shm/corr.bin]
//                        [--gpu_device 0]
//
// The defaults are the reference's. Sizes are checked from the files before anything is read; the inputs are read
// into pinned memory. One line on stderr reports the sizes, the device time (the correlate call, CUDA events) and the
// total time. Exit status 0 on success, 1 on a refused input or a failed read, write or device call, 2 on bad options.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <filesystem>
#include <fstream>
#include <string>
#include <system_error>

#include "srtb_b200.h"

namespace {

struct options {
  std::string in_1 = "pol_1.bin", in_2 = "pol_2.bin", out = "/dev/shm/corr.bin";
  int gpu = 0;
};

int usage(const char* argv0) {
  std::fprintf(stderr,
               "usage: %s [--input_file_1 FILE] [--input_file_2 FILE] [--output_file FILE] [--gpu_device N]\n"
               "defaults: pol_1.bin, pol_2.bin, /dev/shm/corr.bin, device 0\n",
               argv0);
  return 2;
}

int error(const std::string& msg) {
  std::fprintf(stderr, "[correlator] error: %s\n", msg.c_str());
  return 1;
}

bool read_exact(const std::string& path, void* dst, size_t bytes) {
  std::ifstream f(path, std::ios::in | std::ios::binary);
  if (!f) return false;
  f.read(static_cast<char*>(dst), static_cast<std::streamsize>(bytes));
  return static_cast<size_t>(f.gcount()) == bytes;
}

// host and device buffers of one run, released on every exit path
struct buffers {
  unsigned char* h_in[2] = {nullptr, nullptr};
  float* h_out = nullptr;
  void* d_in[2] = {nullptr, nullptr};
  float* d_out = nullptr;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  srtb_b200_ctx* ctx = nullptr;
  ~buffers() {
    if (stream) cudaStreamSynchronize(stream);
    srtb_b200_ctx_destroy(ctx);
    for (auto* p : h_in) cudaFreeHost(p);
    cudaFreeHost(h_out);
    for (auto* p : d_in) cudaFree(p);
    cudaFree(d_out);
    for (auto e : ev)
      if (e) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
  }
};

#define CUDA_OR_FAIL(call)                                                                              \
  do {                                                                                                  \
    const cudaError_t e_ = (call);                                                                      \
    if (e_ != cudaSuccess) return error(std::string(#call) + ": " + cudaGetErrorString(e_));            \
  } while (0)

}  // namespace

int main(int argc, char** argv) {
  const auto t0 = std::chrono::steady_clock::now();
  options o;
  for (int i = 1; i < argc; i++) {
    const std::string k = argv[i];
    if (k == "-h" || k == "--help") {
      usage(argv[0]);
      return 0;
    }
    if (i + 1 >= argc) return usage(argv[0]);
    const std::string v = argv[++i];
    if (k == "--input_file_1") o.in_1 = v;
    else if (k == "--input_file_2") o.in_2 = v;
    else if (k == "--output_file") o.out = v;
    else if (k == "--gpu_device") {
      char* end = nullptr;
      const long d = std::strtol(v.c_str(), &end, 10);
      if (v.empty() || *end || d < 0) return usage(argv[0]);
      o.gpu = static_cast<int>(d);
    } else {
      std::fprintf(stderr, "[correlator] unknown option %s\n", k.c_str());
      return usage(argv[0]);
    }
  }

  // sizes, before anything is read: the rules of srtb_b200_correlate
  size_t size[2];
  const std::string* path[2] = {&o.in_1, &o.in_2};
  for (int s = 0; s < 2; s++) {
    std::error_code ec;
    size[s] = std::filesystem::file_size(*path[s], ec);
    if (ec) return error("cannot read the size of " + *path[s] + ": " + ec.message());
  }
  const size_t input_size = std::min(size[0], size[1]);
  const size_t complex_count = input_size / 2, real_count = 2 * complex_count;
  if (input_size < 2) return error("input_size must be at least 2 bytes, got " + std::to_string(input_size));
  if (real_count & (real_count - 1)) return error("[fft] n must be a power of 2, got " + std::to_string(real_count));
  if (real_count > ((size_t)1 << 31))
    return error("real_count " + std::to_string(real_count) + " above 2^31 samples not supported");

  buffers b;
  CUDA_OR_FAIL(cudaSetDevice(o.gpu));
  CUDA_OR_FAIL(cudaStreamCreateWithFlags(&b.stream, cudaStreamNonBlocking));
  for (int s = 0; s < 2; s++) {
    // real_count bytes of each file: for an odd input_size the reference reads one byte more than its buffer holds
    CUDA_OR_FAIL(cudaMallocHost(reinterpret_cast<void**>(&b.h_in[s]), real_count));
    if (!read_exact(*path[s], b.h_in[s], real_count)) return error("short read from " + *path[s]);
  }
  CUDA_OR_FAIL(cudaMallocHost(reinterpret_cast<void**>(&b.h_out), complex_count * sizeof(float)));
  for (auto& p : b.d_in) CUDA_OR_FAIL(cudaMalloc(&p, real_count));
  CUDA_OR_FAIL(cudaMalloc(reinterpret_cast<void**>(&b.d_out), complex_count * sizeof(float)));
  for (auto& e : b.ev) CUDA_OR_FAIL(cudaEventCreate(&e));
  if (int rc = srtb_b200_ctx_create(o.gpu, b.stream, &b.ctx))
    return error("ctx_create (" + std::to_string(rc) + "): " + srtb_b200_last_error(nullptr));

  for (int s = 0; s < 2; s++)
    CUDA_OR_FAIL(cudaMemcpyAsync(b.d_in[s], b.h_in[s], real_count, cudaMemcpyHostToDevice, b.stream));
  CUDA_OR_FAIL(cudaEventRecord(b.ev[0], b.stream));
  if (int rc = srtb_b200_correlate(b.ctx, b.d_in[0], b.d_in[1], input_size, b.d_out))
    return error("correlate (" + std::to_string(rc) + "): " + srtb_b200_last_error(b.ctx));
  CUDA_OR_FAIL(cudaEventRecord(b.ev[1], b.stream));
  CUDA_OR_FAIL(cudaMemcpyAsync(b.h_out, b.d_out, complex_count * sizeof(float), cudaMemcpyDeviceToHost, b.stream));
  CUDA_OR_FAIL(cudaStreamSynchronize(b.stream));
  float device_ms = 0.f;
  CUDA_OR_FAIL(cudaEventElapsedTime(&device_ms, b.ev[0], b.ev[1]));

  {
    std::ofstream f(o.out, std::ios::out | std::ios::binary | std::ios::trunc);
    f.write(reinterpret_cast<const char*>(b.h_out), static_cast<std::streamsize>(complex_count * sizeof(float)));
    f.close();
    if (!f) return error("cannot write " + o.out);
  }
  const double total_ms =
      std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  std::fprintf(stderr,
               "[correlator] %s: %zu bytes, %s: %zu bytes -> input_size %zu, %zu floats to %s; device %.3f ms, "
               "total %.3f ms\n",
               o.in_1.c_str(), size[0], o.in_2.c_str(), size[1], input_size, complex_count, o.out.c_str(),
               (double)device_ms, total_ms);
  return 0;
}
