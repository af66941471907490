// src/correlator.cpp — `srtb_b200_correlator`, the basic baseband correlator (the reference's
// userspace/src/correlator.cpp): reads two recordings of unsigned 8-bit samples (two polarisations or two antennas),
// forms their cross spectrum and writes the magnitude of the cross-correlation, complex_count = min(size) / 2 raw
// float32 values, as the reference writes them. The device work is one srtb_b200_correlate call.
//
//   srtb_b200_correlator [--input_file_1 pol_1.bin] [--input_file_2 pol_2.bin] [--output_file /dev/shm/corr.bin]
//                        [--gpu_device 0] [--segment_size Ls [--input_bits 8]]
//
// The defaults are the reference's. Sizes are checked from the files before anything is read; the inputs are read
// into pinned memory. One line on stderr reports the sizes, the device time (the correlate call, CUDA events) and the
// total time. Exit status 0 on success, 1 on a refused input or a failed read, write or device call, 2 on bad options.
//
// --segment_size Ls selects the integrating mode (srtb_b200_correlate_accumulate / _finish): each file holds
// floor(size * 8 / |bits|) samples of --input_bits 1, 2, 4, 8 (the default) or -8; K = floor(min(samples) / Ls)
// segments of Ls samples are averaged, and the tail beyond K Ls samples is dropped. Both files are read in chunks of
// max(1, 2^26 / Ls) segments, each chunk one accumulate call (reset on the first), then one finish call writes
// Ms = Ls / 2 raw float32 values, so device memory stays bounded whatever the file size. The next chunk is read while
// the device works on the previous one. The stderr line adds bits, Ls, K, the dropped samples of each file and the
// read time; the device time is then the sum of the accumulate and finish calls. --input_bits other than 8 without
// --segment_size is a usage error.
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
  bool segments = false;  // --segment_size given: the integrating mode
  size_t segment_size = 0;
  int bits = 8;
};

int usage(const char* argv0) {
  std::fprintf(stderr,
               "usage: %s [--input_file_1 FILE] [--input_file_2 FILE] [--output_file FILE] [--gpu_device N]\n"
               "          [--segment_size Ls [--input_bits 1|2|4|8|-8]]\n"
               "defaults: pol_1.bin, pol_2.bin, /dev/shm/corr.bin, device 0, whole-file mode, 8-bit samples\n",
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
// (the integrating mode: h_in[2 slot + input] double-buffers the chunks, ev[2 slot], ev[2 slot + 1] bracket the
// accumulate call of the slot's chunk and ev[4], ev[5] the finish call)
struct buffers {
  unsigned char* h_in[4] = {nullptr, nullptr, nullptr, nullptr};
  float* h_out = nullptr;
  void* d_in[2] = {nullptr, nullptr};
  void* d_acc = nullptr;
  float* d_out = nullptr;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[6] = {};
  srtb_b200_ctx* ctx = nullptr;
  ~buffers() {
    if (stream) cudaStreamSynchronize(stream);
    srtb_b200_ctx_destroy(ctx);
    for (auto* p : h_in) cudaFreeHost(p);
    cudaFreeHost(h_out);
    for (auto* p : d_in) cudaFree(p);
    cudaFree(d_acc);
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

bool write_out(const std::string& path, const float* v, size_t n) {
  std::ofstream f(path, std::ios::out | std::ios::binary | std::ios::trunc);
  f.write(reinterpret_cast<const char*>(v), static_cast<std::streamsize>(n * sizeof(float)));
  f.close();
  return static_cast<bool>(f);
}

double ms_since(std::chrono::steady_clock::time_point t) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count();
}

// the integrating mode, from the two file sizes
int run_segments(const options& o, const size_t size[2], std::chrono::steady_clock::time_point t0) {
  const size_t Ls = o.segment_size, Ms = Ls / 2;
  const size_t abits = o.bits < 0 ? -o.bits : o.bits;
  // srtb_b200_correlate_accumulate's rule and message, checked before anything is read
  if ((Ls & (Ls - 1)) || Ls < 16 || Ls > ((size_t)1 << 30))
    return error("correlate_accumulate: segment_size must be a power of two from 16 to 2^30, got " + std::to_string(Ls));
  size_t samples[2];
  for (int s = 0; s < 2; s++) samples[s] = size[s] * (8 / abits);  // floor(size 8 / |bits|)
  const size_t K = std::min(samples[0], samples[1]) / Ls;
  if (K == 0)
    return error("no complete segment of " + std::to_string(Ls) + " samples: " + std::to_string(samples[0]) + " and " +
                 std::to_string(samples[1]) + " samples");
  const size_t chunk = std::max<size_t>(1, ((size_t)1 << 26) / Ls);  // segments per accumulate call
  const size_t seg_bytes = Ls * abits / 8, chunks = (K + chunk - 1) / chunk;
  const size_t chunk_bytes = std::min(chunk, K) * seg_bytes;

  buffers b;
  CUDA_OR_FAIL(cudaSetDevice(o.gpu));
  CUDA_OR_FAIL(cudaStreamCreateWithFlags(&b.stream, cudaStreamNonBlocking));
  const int slots = chunks > 1 ? 2 : 1;
  for (int i = 0; i < 2 * slots; i++) CUDA_OR_FAIL(cudaMallocHost(reinterpret_cast<void**>(&b.h_in[i]), chunk_bytes));
  CUDA_OR_FAIL(cudaMallocHost(reinterpret_cast<void**>(&b.h_out), Ms * sizeof(float)));
  for (auto& p : b.d_in) CUDA_OR_FAIL(cudaMalloc(&p, chunk_bytes));
  CUDA_OR_FAIL(cudaMalloc(&b.d_acc, Ms * 2 * sizeof(double)));
  CUDA_OR_FAIL(cudaMalloc(reinterpret_cast<void**>(&b.d_out), Ms * sizeof(float)));
  for (auto& e : b.ev) CUDA_OR_FAIL(cudaEventCreate(&e));
  if (int rc = srtb_b200_ctx_create(o.gpu, b.stream, &b.ctx))
    return error("ctx_create (" + std::to_string(rc) + "): " + srtb_b200_last_error(nullptr));

  std::ifstream f[2] = {std::ifstream(o.in_1, std::ios::in | std::ios::binary),
                        std::ifstream(o.in_2, std::ios::in | std::ios::binary)};
  const std::string* path[2] = {&o.in_1, &o.in_2};
  double read_ms = 0.0;
  float device_ms = 0.f;
  bool pending[2] = {false, false};
  // adds the device time of the slot's last chunk once it is done; its host buffers are then free again
  auto drain = [&](int slot) -> int {
    if (!pending[slot]) return 0;
    float ms = 0.f;
    CUDA_OR_FAIL(cudaEventSynchronize(b.ev[2 * slot + 1]));
    CUDA_OR_FAIL(cudaEventElapsedTime(&ms, b.ev[2 * slot], b.ev[2 * slot + 1]));
    device_ms += ms;
    pending[slot] = false;
    return 0;
  };
  for (size_t c = 0, done = 0; c < chunks; c++) {
    const int slot = (int)(c % slots);
    const size_t n = std::min(chunk, K - done), bytes = n * seg_bytes;
    if (int rc = drain(slot)) return rc;
    const auto r0 = std::chrono::steady_clock::now();
    for (int s = 0; s < 2; s++) {
      f[s].read(reinterpret_cast<char*>(b.h_in[2 * slot + s]), static_cast<std::streamsize>(bytes));
      if (!f[s] || static_cast<size_t>(f[s].gcount()) != bytes) return error("short read from " + *path[s]);
    }
    read_ms += ms_since(r0);
    for (int s = 0; s < 2; s++)
      CUDA_OR_FAIL(cudaMemcpyAsync(b.d_in[s], b.h_in[2 * slot + s], bytes, cudaMemcpyHostToDevice, b.stream));
    CUDA_OR_FAIL(cudaEventRecord(b.ev[2 * slot], b.stream));
    if (int rc = srtb_b200_correlate_accumulate(b.ctx, b.d_in[0], b.d_in[1], o.bits, Ls, n, b.d_acc, c == 0))
      return error("correlate_accumulate (" + std::to_string(rc) + "): " + srtb_b200_last_error(b.ctx));
    CUDA_OR_FAIL(cudaEventRecord(b.ev[2 * slot + 1], b.stream));
    pending[slot] = true;
    done += n;
  }
  CUDA_OR_FAIL(cudaEventRecord(b.ev[4], b.stream));
  if (int rc = srtb_b200_correlate_finish(b.ctx, b.d_acc, Ls, K, b.d_out))
    return error("correlate_finish (" + std::to_string(rc) + "): " + srtb_b200_last_error(b.ctx));
  CUDA_OR_FAIL(cudaEventRecord(b.ev[5], b.stream));
  CUDA_OR_FAIL(cudaMemcpyAsync(b.h_out, b.d_out, Ms * sizeof(float), cudaMemcpyDeviceToHost, b.stream));
  CUDA_OR_FAIL(cudaStreamSynchronize(b.stream));
  for (int slot = 0; slot < slots; slot++)
    if (int rc = drain(slot)) return rc;
  float finish_ms = 0.f;
  CUDA_OR_FAIL(cudaEventElapsedTime(&finish_ms, b.ev[4], b.ev[5]));
  device_ms += finish_ms;

  if (!write_out(o.out, b.h_out, Ms)) return error("cannot write " + o.out);
  std::fprintf(stderr,
               "[correlator] %s: %zu bytes, %s: %zu bytes, bits %d, segment_size %zu -> K %zu segments in %zu chunks, "
               "dropped %zu and %zu samples at the tail, %zu floats to %s; read %.3f ms, device %.3f ms, "
               "total %.3f ms\n",
               o.in_1.c_str(), size[0], o.in_2.c_str(), size[1], o.bits, Ls, K, chunks, samples[0] - K * Ls,
               samples[1] - K * Ls, Ms, o.out.c_str(), read_ms, (double)device_ms, ms_since(t0));
  return 0;
}

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
    } else if (k == "--segment_size") {
      char* end = nullptr;
      const unsigned long long n = std::strtoull(v.c_str(), &end, 10);
      if (v.empty() || *end || v[0] == '-') return usage(argv[0]);
      o.segments = true;
      o.segment_size = static_cast<size_t>(n);
    } else if (k == "--input_bits") {
      char* end = nullptr;
      const long n = std::strtol(v.c_str(), &end, 10);
      if (v.empty() || *end || (n != 1 && n != 2 && n != 4 && n != 8 && n != -8)) return usage(argv[0]);
      o.bits = static_cast<int>(n);
    } else {
      std::fprintf(stderr, "[correlator] unknown option %s\n", k.c_str());
      return usage(argv[0]);
    }
  }
  if (o.bits != 8 && !o.segments) {
    std::fprintf(stderr, "[correlator] --input_bits %d needs --segment_size\n", o.bits);
    return usage(argv[0]);
  }

  // sizes, before anything is read: the rules of srtb_b200_correlate
  size_t size[2];
  const std::string* path[2] = {&o.in_1, &o.in_2};
  for (int s = 0; s < 2; s++) {
    std::error_code ec;
    size[s] = std::filesystem::file_size(*path[s], ec);
    if (ec) return error("cannot read the size of " + *path[s] + ": " + ec.message());
  }
  if (o.segments) return run_segments(o, size, t0);
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
