// =============================================================================
// srtb_oracle.cpp — CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT CODE)
//
// A plain C++/OpenMP restatement of the reference's baseband -> single-pulse
// chain (fxzjshm/simple-radio-telescope-backend @ 49fac3ae), operator by
// operator, with the reference's arithmetic types and rounding points.
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
// --impl reference legs may load this library; the product path
// (libsrtb_b200.so) never links or calls it.
//
// Parity pinning: the restatement is checked against every known-answer vector
// the reference's own tests hold for this path (tests/test_oracle_golden.py):
//   unpack KATs      userspace/tests/test-unpack.cpp:65-67,84-86,104-106,123-125,146-199
//   hamming(16)      userspace/tests/test-fft_window.cpp:39-48
//   manual RFI zap   userspace/tests/test-rfi_mitigation.cpp:28-31,52-70
//   FFT              cross-checked against float64 numpy.fft (the reference pins its
//                    FFT only against FFTW, tests/test-naive_fft.cpp:148-157)
// and, when /root/reference is present, against the reference headers themselves
// compiled through a host SYCL shim (oracle/ref_shim -> oracle/_ref/libsrtb_ref.so).
// tests/test_oracle_vs_ref.py: bit-exact for unpack / window / FFT / chirp / s1 values / SK rows,
// masks and counts identical off the threshold border). Stages the reference never tests
// (s1, SK, chirp values, waterfall layout, detect) are pinned by that build; see DESIGN.md section 4.
//
// Build: make -C oracle   (g++ -O2 -fopenmp -ffp-contract=off: the reference is built
// with -fno-fast-math and contraction only inside one expression,
// userspace/CMakeLists.txt:188-193; we compute unfused.)
//
// S/ = /root/reference/userspace/include/srtb/ in the citations below.
// =============================================================================
#include <algorithm>
#include <cmath>
#include <complex>
#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#if defined(_OPENMP)
#include <omp.h>
#endif

namespace {

using real = float;  // S/math.hpp:44
struct cf {
  float re, im;
};

// SyclCPLX operator* for finite operands: (ac - bd, ad + bc), four separately rounded
// products (U/3rdparty/SyclCPLX/include/sycl_ext_complex.hpp:569-623; SURVEY q11).
static inline cf cmul(cf a, cf b) {
  const float ac = a.re * b.re, bd = a.im * b.im, ad = a.re * b.im, bc = a.im * b.re;
  return cf{ac - bd, ad + bc};
}
static inline cf cadd(cf a, cf b) { return cf{a.re + b.re, a.im + b.im}; }
static inline cf csub(cf a, cf b) { return cf{a.re - b.re, a.im - b.im}; }
static inline cf cconj(cf a) { return cf{a.re, -a.im}; }
static inline float cnorm(cf a) { return a.re * a.re + a.im * a.im; }  // S/math.hpp:58-66

// Fixed-order pairwise fp32 sum (the reference's order is device dependent,
// P/algorithm/buffer_algorithms.hpp:88-131; SURVEY appendix B says: fixed pairwise).
template <typename F>
static float pairwise_sum(size_t lo, size_t hi, const F& f) {
  const size_t n = hi - lo;
  if (n <= 64) {
    float s = 0.0f;
    for (size_t i = lo; i < hi; i++) s += f(i);
    return s;
  }
  const size_t mid = lo + n / 2;
  return pairwise_sum(lo, mid, f) + pairwise_sum(mid, hi, f);
}

template <typename F>
static float parallel_pairwise_sum(size_t n, const F& f) {
  // split into 256 fixed chunks (independent of thread count) -> deterministic
  const size_t chunks = 256;
  if (n < chunks * 1024) return pairwise_sum(0, n, f);
  std::vector<float> part(chunks);
#pragma omp parallel for schedule(static)
  for (long c = 0; c < (long)chunks; c++) {
    const size_t lo = n * (size_t)c / chunks, hi = n * (size_t)(c + 1) / chunks;
    part[c] = pairwise_sum(lo, hi, f);
  }
  return pairwise_sum(0, chunks, [&](size_t i) { return part[i]; });
}

// ---------------------------------------------------------------------------
// window  (S/fft/fft_window.hpp:27-50 cosine_sum_window, :91-106 functor,
//          :112-123 iterator: x = float(i) / (n - 1))
// 0 = rectangle (default, :83), 1 = hann {0.5,0.5} (:52-59), 2 = hamming {25/46,21/46} (:61-68)
// ---------------------------------------------------------------------------
static inline float window_value(int window, size_t i, size_t n) {
  if (window == 0) return 1.0f;
  float a[2];
  if (window == 1) {
    a[0] = 0.5f;
    a[1] = 0.5f;
  } else {
    a[0] = (float)(25.0 / 46.0);
    a[1] = (float)(21.0 / 46.0);
  }
  const float x = static_cast<float>(i) / static_cast<float>(n - 1);  // float / size_t
  float ret = 0;
  for (size_t k = 0; k < 2; k++) {
    const float sign = ((k & 1) == 0) ? 1.0f : -1.0f;
    // `2 * M_PI * k * x` is double, sycl::cos(double); ret += (float*float)*double
    ret = (float)((double)ret + (double)(sign * a[k]) * std::cos(2 * M_PI * (double)k * (double)x));
  }
  return ret;
}

}  // namespace

extern "C" {

float srtb_oracle_window(int window, size_t i, size_t n) { return window_value(window, i, n); }

// ---------------------------------------------------------------------------
// unpack "simple"  (S/unpack.hpp:43-156 item functions, :171-197 driver;
// dispatch on bits S/pipeline/unpack_pipe.hpp:72-127)
// out_count = in_bytes * 8 / |bits|   (unpack_pipe.hpp:49-51)
// returns 0, or -1 for unsupported bits (the reference throws, :123-127)
// ---------------------------------------------------------------------------
int srtb_oracle_unpack(const void* in_, size_t out_count, int bits, int window, float* out) {
  const uint8_t* in = static_cast<const uint8_t*>(in_);
  const size_t n = out_count;
  if (bits == 1 || bits == 2 || bits == 4) {
    const int count = 8 / bits;
    const unsigned mask = (1u << bits) - 1u;
    const size_t nbytes = out_count * (size_t)bits / 8;
#pragma omp parallel for schedule(static)
    for (long xx = 0; xx < (long)nbytes; xx++) {
      const size_t x = (size_t)xx;
      const unsigned v = in[x];
      for (int i = 0; i < count; i++) {
        // MSB first: (in & (mask << (8-b) >> i*b)) >> ((count-i-1)*b)   (unpack.hpp:52-74)
        const unsigned val = (v >> ((count - i - 1) * bits)) & mask;
        const size_t pos = (size_t)count * x + (size_t)i;
        out[pos] = static_cast<float>(val) * window_value(window, pos, n);
      }
    }
    return 0;
  }
#define SRTB_ORACLE_CAST(T)                                                        \
  {                                                                                \
    const T* p = static_cast<const T*>(in_);                                       \
    _Pragma("omp parallel for schedule(static)") for (long x = 0; x < (long)n; x++) \
        out[x] = static_cast<float>(p[x]) * window_value(window, (size_t)x, n);    \
    return 0;                                                                      \
  }
  if (bits == 8) SRTB_ORACLE_CAST(uint8_t)
  if (bits == -8) SRTB_ORACLE_CAST(int8_t)
  if (bits == 16) SRTB_ORACLE_CAST(uint16_t)
  if (bits == -16) SRTB_ORACLE_CAST(int16_t)
  if (bits == 32) SRTB_ORACLE_CAST(float)
  if (bits == 64) SRTB_ORACLE_CAST(double)
  return -1;
}

// "1 2 1 2" interleave (S/unpack.hpp:221-244), bits in {8,-8,16,-16,32,64}
// (S/pipeline/unpack_pipe.hpp:186-236). out_count = per-stream count.
int srtb_oracle_unpack_interleaved_2(const void* in_, size_t out_count, int bits, int window,
                                     float* out1, float* out2) {
  const size_t n = out_count;
#define SRTB_ORACLE_IL2(T)                                                 \
  {                                                                        \
    const T* p = static_cast<const T*>(in_);                               \
    _Pragma("omp parallel for schedule(static)") for (long xx = 0; xx < (long)n; xx++) { \
      const size_t x = (size_t)xx;                                         \
      const float w = window_value(window, x, n);                          \
      out1[x] = static_cast<float>(p[2 * x]) * w;                          \
      out2[x] = static_cast<float>(p[2 * x + 1]) * w;                      \
    }                                                                      \
    return 0;                                                              \
  }
  if (bits == 8) SRTB_ORACLE_IL2(uint8_t)
  if (bits == -8) SRTB_ORACLE_IL2(int8_t)
  if (bits == 16) SRTB_ORACLE_IL2(uint16_t)
  if (bits == -16) SRTB_ORACLE_IL2(int16_t)
  if (bits == 32) SRTB_ORACLE_IL2(float)
  if (bits == 64) SRTB_ORACLE_IL2(double)
  return -1;
}

// naocpsr_snap1 "1 1 2 2" int8 (S/unpack.hpp:255-283): work item x < out_count/2
int srtb_oracle_unpack_snap1(const void* in_, size_t out_count, int window, float* out1,
                             float* out2) {
  const int8_t* in = static_cast<const int8_t*>(in_);
  const size_t n = out_count;
#pragma omp parallel for schedule(static)
  for (long xx = 0; xx < (long)(n / 2); xx++) {
    const size_t x = (size_t)xx;
    out1[2 * x] = static_cast<float>(in[4 * x]) * window_value(window, 2 * x, n);
    out1[2 * x + 1] = static_cast<float>(in[4 * x + 1]) * window_value(window, 2 * x + 1, n);
    out2[2 * x] = static_cast<float>(in[4 * x + 2]) * window_value(window, 2 * x, n);
    out2[2 * x + 1] = static_cast<float>(in[4 * x + 3]) * window_value(window, 2 * x + 1, n);
  }
  return 0;
}

// gznupsr_a1: 4-sample words round-robin to `streams` (4 or 2) outputs
// (S/unpack.hpp:293-369). The 4-output variant computes float(int(in) ^ 0x80) on an
// int8 input (:315-316) — integer promotion happens BEFORE the xor, so -128 -> -256,
// -1 -> -129, 0 -> 128, 127 -> 255; the 2-output variant has no xor (:356-357).
int srtb_oracle_unpack_gznupsr_a1(const void* in_, size_t out_count, int streams, int window,
                                  float* const* out) {
  const int8_t* in = static_cast<const int8_t*>(in_);
  const size_t n = out_count;
  if (streams != 2 && streams != 4) return -1;
#pragma omp parallel for schedule(static)
  for (long xx = 0; xx < (long)(n / 4); xx++) {
    const size_t x = (size_t)xx;
    for (int i = 0; i < streams; i++)
      for (int j = 0; j < 4; j++) {
        const int8_t s = in[(size_t)streams * 4 * x + (size_t)i * 4 + (size_t)j];
        const float v = (streams == 4) ? static_cast<float>(static_cast<int>(s) ^ 0x80)
                                       : static_cast<float>(s);
        out[i][4 * x + j] = v * window_value(window, 4 * x + j, n);
      }
  }
  return 0;
}

// ---------------------------------------------------------------------------
// naive radix-2 FFT (S/fft/naive_fft.hpp): bit_reverse_swap :93-106, butterfly
// :117-145 (theta in f32, cos/sin per butterfly), driver :155-176, no normalisation.
// direction +1 = forward (e^{-i..}), -1 = backward.
// ---------------------------------------------------------------------------
static void naive_c2c(cf* x, unsigned k, int direction) {
  const size_t n = (size_t)1 << k;
  // bit reverse swap (in place: input == output, i <= j swap)
#pragma omp parallel for schedule(static)
  for (long ii = 0; ii < (long)n; ii++) {
    const size_t i = (size_t)ii;
    size_t j = 0, t = i;
    for (unsigned b = 0; b < k; b++) {
      j = (j << 1) | (t & 1);
      t >>= 1;
    }
    if (i < j) std::swap(x[i], x[j]);
  }
  for (unsigned m = 0; m < k; ++m) {
    const size_t butterfly_size = (size_t)1 << (m + 1);
#pragma omp parallel for schedule(static)
    for (long ii = 0; ii < (long)(n / 2); ii++) {
      const size_t i = (size_t)ii;
      const size_t group = i >> m;
      const size_t local = i - (group << m);
      const size_t xi = group * butterfly_size + local;
      const size_t yi = xi + (butterfly_size / 2);
      // -T{2.0*M_PI} * local / size * direction, all in f32, left to right (:136-137)
      const float theta = ((-static_cast<float>(2.0 * M_PI) * static_cast<float>(local)) /
                           static_cast<float>(butterfly_size)) *
                          static_cast<float>(direction);
      const cf w{std::cos(theta), std::sin(theta)};
      const cf cx = x[xi], cy = x[yi];
      const cf wy = cmul(w, cy);
      x[xi] = cadd(cx, wy);
      x[yi] = csub(cx, wy);
    }
  }
}

void srtb_oracle_fft_c2c(float* x, size_t n, int direction) {
  unsigned k = 0;
  while (((size_t)1 << k) < n) k++;
  naive_c2c(reinterpret_cast<cf*>(x), k, direction);
}

// R2C in place on N+2 floats (S/fft/naive_fft.hpp:221-261): N/2-point C2C on the packed
// pairs, then the split post-process for k = 0..N/4; writes bins 0..N/2 inclusive.
void srtb_oracle_fft_r2c(float* inout, size_t n_real) {
  unsigned k = 0;
  while (((size_t)1 << k) < n_real) k++;
  const size_t N = n_real / 2;
  cf* H = reinterpret_cast<cf*>(inout);
  naive_c2c(H, k - 1, +1);
#pragma omp parallel for schedule(static)
  for (long kk = 0; kk < (long)(N / 2 + 1); kk++) {
    const size_t kx = (size_t)kk;
    const cf H_k = H[kx];
    const cf H_N_k = (kx == 0) ? H[0] : H[N - kx];
    const cf Hc = cconj(H_N_k);
    const cf s = cadd(H_k, Hc);
    const cf F_k{s.re / 2.0f, s.im / 2.0f};
    const cf d = csub(H_k, Hc);
    const cf mhalf_i{-0.0f / 2.0f, -1.0f / 2.0f};  // -C{0,1} / T{2}
    const cf G_k = cmul(d, mhalf_i);
    const cf F_N_k = cconj(F_k), G_N_k = cconj(G_k);
    const float theta_k = (-static_cast<float>(M_PI) * static_cast<float>(kx)) / static_cast<float>(N);
    const float w_re = std::cos(theta_k), w_im = std::sin(theta_k);
    const cf w_k{w_re, w_im}, w_N_k{-w_re, w_im};
    const cf X_k = cadd(F_k, cmul(G_k, w_k));
    const cf X_N_k = cadd(F_N_k, cmul(G_N_k, w_N_k));
    H[kx] = X_k;
    H[N - kx] = X_N_k;
  }
}

// waterfall FFT: batch independent backward C2C of length L on contiguous rows
// (S/pipeline/fft_pipe.hpp:313-371; naive fallback loops the batch,
//  S/fft/naive_fft_wrapper.hpp:88-91)
void srtb_oracle_watfft(float* x, size_t length, size_t batch) {
  unsigned k = 0;
  while (((size_t)1 << k) < length) k++;
  cf* p = reinterpret_cast<cf*>(x);
  // rows in parallel (inner loops are then serial per row)
#pragma omp parallel for schedule(dynamic)
  for (long b = 0; b < (long)batch; b++) {
    cf* row = p + (size_t)b * length;
    const size_t n = length;
    for (size_t i = 0; i < n; i++) {
      size_t j = 0, t = i;
      for (unsigned bb = 0; bb < k; bb++) {
        j = (j << 1) | (t & 1);
        t >>= 1;
      }
      if (i < j) std::swap(row[i], row[j]);
    }
    for (unsigned m = 0; m < k; ++m) {
      const size_t bs = (size_t)1 << (m + 1);
      for (size_t i = 0; i < n / 2; i++) {
        const size_t group = i >> m, local = i - (group << m);
        const size_t xi = group * bs + local, yi = xi + bs / 2;
        const float theta = ((-static_cast<float>(2.0 * M_PI) * static_cast<float>(local)) /
                             static_cast<float>(bs)) *
                            static_cast<float>(-1);
        const cf w{std::cos(theta), std::sin(theta)};
        const cf cx = row[xi], cy = row[yi];
        const cf wy = cmul(w, cy);
        row[xi] = cadd(cx, wy);
        row[yi] = csub(cx, wy);
      }
    }
  }
}

// ---------------------------------------------------------------------------
// RFI stage 1 (S/pipeline/rfi_mitigation_pipe.hpp:43-101)
// mean of |X|^2 (map_average, S/algorithm/map_reduce.hpp:84-91: sum / float(count)),
// coef = pow(float(Nc)*float(Nc)/float(C), -0.5) (:61-65), zap or normalise (:66-79).
// Returns the mean through *mean_out. zap mask written if mask != NULL.
// ---------------------------------------------------------------------------
float srtb_oracle_norm_coefficient(size_t in_count, size_t channel_count) {
  return static_cast<float>(std::pow(
      static_cast<float>(in_count) * static_cast<float>(in_count) / static_cast<float>(channel_count),
      -0.5));
}

void srtb_oracle_rfi_s1_average(float* x_, size_t in_count, float threshold, size_t channel_count,
                                float* mean_out, uint8_t* mask) {
  cf* x = reinterpret_cast<cf*>(x_);
  const float sum = parallel_pairwise_sum(in_count, [&](size_t i) { return cnorm(x[i]); });
  const float norm_avg = sum / static_cast<float>(in_count);
  const float coef = srtb_oracle_norm_coefficient(in_count, channel_count);
  if (mean_out) *mean_out = norm_avg;
#pragma omp parallel for schedule(static)
  for (long ii = 0; ii < (long)in_count; ii++) {
    const size_t i = (size_t)ii;
    const cf in = x[i];
    const float val = cnorm(in);
    if (val > threshold * norm_avg) {
      x[i] = cf{0, 0};
      if (mask) mask[i] = 1;
    } else {
      x[i] = cf{in.re * coef, in.im * coef};
      if (mask) mask[i] = 0;
    }
  }
}

// "a-b, c-d" parser (S/spectrum/rfi_mitigation.hpp:64-88): split on ',', then on '-',
// token_compress_on, std::stod each. Returns number of pairs written (<= max_pairs).
size_t srtb_oracle_eval_rfi_ranges(const char* list, float* pairs, size_t max_pairs) {
  auto split = [](const std::string& s, char sep) {
    // boost::split with token_compress_on: adjacent separators merge, but leading /
    // trailing separators still yield empty tokens at the ends.
    std::vector<std::string> out;
    std::string cur;
    bool last_sep = false;
    for (char c : s) {
      if (c == sep) {
        if (!last_sep) {
          out.push_back(cur);
          cur.clear();
        }
        last_sep = true;
      } else {
        cur.push_back(c);
        last_sep = false;
      }
    }
    out.push_back(cur);
    return out;
  };
  size_t n = 0;
  const std::string s(list);
  for (const std::string& str : split(s, ',')) {
    const std::vector<std::string> nums = split(str, '-');
    if (nums.size() != 2) continue;  // reference logs a warning (:76-78)
    float f1, f2;
    try {
      f1 = static_cast<float>(std::stod(nums[0]));
      f2 = static_cast<float>(std::stod(nums[1]));
    } catch (...) {
      continue;  // reference would throw std::invalid_argument from stod
    }
    if (n < max_pairs) {
      pairs[2 * n] = f1;
      pairs[2 * n + 1] = f2;
    }
    n++;
  }
  return n;
}

// MHz range -> inclusive bin range (S/spectrum/rfi_mitigation.hpp:102-143).
// Returns 1 and fills lo/hi if the range is applied, 0 if rejected (out of bounds).
int srtb_oracle_rfi_range_to_bins(float f1, float f2, float freq_low, float bandwidth,
                                  size_t in_count, size_t* lo, size_t* hi) {
  const bool bw_sign = std::signbit(bandwidth);
  const bool r_sign = std::signbit(f2 - f1);
  if (bw_sign != r_sign) std::swap(f1, f2);
  const float a = std::round((f1 - freq_low) / bandwidth * static_cast<float>(in_count - 1));
  const float b = std::round((f2 - freq_low) / bandwidth * static_cast<float>(in_count - 1));
  // static_cast<size_t>(negative float) is UB in the reference; any sane platform value
  // (0x8000.. on x86-64) fails the `hi < in_count` check, so: reject negatives.
  if (!(a >= 0.0f) || !(b >= 0.0f)) return 0;
  if (a >= 1.8446744e19f || b >= 1.8446744e19f) return 0;
  const size_t l = static_cast<size_t>(a), h = static_cast<size_t>(b);
  if (l <= h && h < in_count) {
    *lo = l;
    *hi = h;
    return 1;
  }
  return 0;
}

size_t srtb_oracle_rfi_manual(float* x_, size_t in_count, float freq_low, float bandwidth,
                              const float* pairs, size_t n_pairs) {
  cf* x = reinterpret_cast<cf*>(x_);
  size_t applied = 0;
  for (size_t r = 0; r < n_pairs; r++) {
    size_t lo, hi;
    if (srtb_oracle_rfi_range_to_bins(pairs[2 * r], pairs[2 * r + 1], freq_low, bandwidth, in_count,
                                      &lo, &hi)) {
      for (size_t i = lo; i <= hi; i++) x[i] = cf{0, 0};
      applied++;
    }
  }
  return applied;
}

// ---------------------------------------------------------------------------
// coherent dedispersion (S/coherent_dedispersion.hpp:133-150 phase_factor_v3,
// :223-237 kernel). f_min, f_c, df, dm arrive as f32 and are promoted (SURVEY q7).
// ---------------------------------------------------------------------------
void srtb_oracle_dedisperse(float* x_, size_t length, float f_min, float f_c_, float df, float dm_) {
  cf* x = reinterpret_cast<cf*>(x_);
  constexpr double D = 4.148808e3;  // :67
  constexpr double D_ = D * 1e6;
#pragma omp parallel for schedule(static)
  for (long ii = 0; ii < (long)length; ii++) {
    const size_t i = (size_t)ii;
    const double f = double{f_min} + double{df} * static_cast<double>(i);
    const double f_c = double{f_c_}, dm = double{dm_};
    const double delta_f = f - f_c;
    const double k = D_ * dm / f * ((delta_f / f_c) * (delta_f / f_c));
    double k_int;
    const float k_frac = static_cast<float>(std::modf(k, &k_int));
    const float delta_phi = -static_cast<float>(2 * M_PI) * k_frac;
    const cf factor{std::cos(delta_phi), std::sin(delta_phi)};
    x[i] = cmul(x[i], factor);
  }
}

// max_delay_time / nsamps_reserved (S/coherent_dedispersion.hpp:76-128)
size_t srtb_oracle_nsamps_reserved(size_t baseband_input_count, size_t channel_count, float freq_low,
                                   float bandwidth, float sample_rate, float dm, int reserve_sample) {
  if (!reserve_sample) return 0;
  constexpr double D = 4.148808e3;
  // dispersion_delay_time<float>(f = low+bw, f_c = low, dm): -D*dm*(1.0/(f*f) - 1.0/(f_c*f_c))
  const float f = freq_low + bandwidth, f_c = freq_low;
  const float delay = static_cast<float>(-D * (double)dm * (1.0 / (double)(f * f) - 1.0 / (double)(f_c * f_c)));
  // 2 * std::round(float * float) is a float expression converted to size_t (:108-110)
  const float minimal_f = 2 * std::round(delay * sample_rate);
  const size_t minimal_reserve_count = static_cast<size_t>(minimal_f < 0 ? 0.0f : minimal_f);
  const size_t per_bin = channel_count * 2;
  const long long refft_total =
      static_cast<long long>(baseband_input_count - minimal_reserve_count) / (long long)per_bin *
      (long long)per_bin;
  const size_t may_reserve = baseband_input_count - (size_t)refft_total;
  if (refft_total > 0) return may_reserve;
  return 0;  // reference also clears config.baseband_reserve_sample (:125)
}

// ---------------------------------------------------------------------------
// RFI stage 2: spectral kurtosis v2 (S/spectrum/rfi_mitigation.hpp:292-341)
// x is [chan_count][time_count], time contiguous. sk_out (may be NULL) receives
// M*s4/(s2*s2) per channel; zap (may be NULL) the decision.
// ---------------------------------------------------------------------------
void srtb_oracle_sk_thresholds(size_t time_count, float sk_threshold, float* lo_, float* hi_) {
  const float M_ = static_cast<float>(time_count);
  float hi = sk_threshold, lo = 2 - sk_threshold;
  if (lo > hi) std::swap(lo, hi);
  *lo_ = lo * ((M_ - 1) / (M_ + 1)) + 1;
  *hi_ = hi * ((M_ - 1) / (M_ + 1)) + 1;
}

void srtb_oracle_rfi_s2(float* x_, size_t time_count, size_t chan_count, float sk_threshold,
                        float* sk_out, uint8_t* zap) {
  cf* x = reinterpret_cast<cf*>(x_);
  float lo, hi;
  srtb_oracle_sk_thresholds(time_count, sk_threshold, &lo, &hi);
#pragma omp parallel for schedule(static)
  for (long cc = 0; cc < (long)chan_count; cc++) {
    const size_t c = (size_t)cc;
    cf* row = x + c * time_count;
    const float s2 = pairwise_sum(0, time_count, [&](size_t t) { return cnorm(row[t]); });
    const float s4 = pairwise_sum(0, time_count, [&](size_t t) {
      const float x2 = cnorm(row[t]);
      return x2 * x2;
    });
    const float sk = static_cast<float>(time_count) * (s4 / (s2 * s2));
    const bool zeroing = (sk > hi || sk < lo);  // NaN -> false (SURVEY q5)
    if (sk_out) sk_out[c] = sk;
    if (zap) zap[c] = zeroing ? 1 : 0;
    if (zeroing)
      for (size_t t = 0; t < time_count; t++) row[t] = cf{0, 0};
  }
}

// ---------------------------------------------------------------------------
// signal detect (S/pipeline/signal_detect_pipe.hpp:252-442, S/signal_detect.hpp:32-72)
// ---------------------------------------------------------------------------
struct srtb_oracle_detect_result {
  uint64_t zero_count;
  uint64_t time_series_count;  // L'
  int32_t detect_enabled;      // zero_count < thr_chan * C
  int32_t n_boxcars;           // entries used below (boxcar 1, 2, 4, ...)
  uint64_t boxcar_length[32];
  uint64_t series_length[32];
  uint64_t signal_count[32];
  float variance[32];   // mean(v^2)
  float threshold[32];  // snr * sqrt(variance)
};

static void count_signal(const float* v, size_t n, float snr, float* var_out, float* thr_out,
                         uint64_t* count_out) {
  const float sum = parallel_pairwise_sum(n, [&](size_t i) { return v[i] * v[i]; });
  const float var = sum / static_cast<float>(n);
  const float thr = static_cast<float>(snr * std::sqrt(var));
  uint64_t cnt = 0;
#pragma omp parallel for reduction(+ : cnt) schedule(static)
  for (long i = 0; i < (long)n; i++)
    if (v[i] > thr) cnt++;
  *var_out = var;
  *thr_out = thr;
  *count_out = cnt;
}

// series_out: caller buffer of 32 * time_count floats; row b holds the series of boxcar
// index b (row 0 = mean-removed time series, row i = boxcar 2^i), valid length
// series_length[i]. Intended values per SURVEY q3 (the reference's buffer reuse bug is
// not reproduced).
void srtb_oracle_signal_detect(const float* x_, size_t time_count, size_t chan_count,
                               size_t time_reserved_count, float snr_threshold,
                               float channel_threshold, size_t max_boxcar_length,
                               srtb_oracle_detect_result* res, float* series_out) {
  const cf* x = reinterpret_cast<const cf*>(x_);
  std::memset(res, 0, sizeof(*res));
  // zero_count: first time sample of every channel (:261-284; SURVEY q4)
  uint64_t zero_count = 0;
  for (size_t c = 0; c < chan_count; c++)
    if (cnorm(x[c * time_count]) == 0) zero_count++;
  res->zero_count = zero_count;
  size_t ts_count;
  if (time_count <= time_reserved_count)
    ts_count = time_count;
  else
    ts_count = time_count - time_reserved_count;
  res->time_series_count = ts_count;
  float* ts = series_out;
  // column sum, ascending channel order, serial per column (:305-316)
#pragma omp parallel for schedule(static)
  for (long jj = 0; jj < (long)ts_count; jj++) {
    const size_t j = (size_t)jj;
    float s = 0;
    for (size_t i = 0; i < chan_count; i++) s += cnorm(x[i * time_count + j]);
    ts[j] = s;
  }
  // baseline removal (:324-334)
  const float avg = parallel_pairwise_sum(ts_count, [&](size_t i) { return ts[i]; }) /
                    static_cast<float>(ts_count);
#pragma omp parallel for schedule(static)
  for (long i = 0; i < (long)ts_count; i++) ts[i] -= avg;

  res->detect_enabled =
      (static_cast<float>(zero_count) < channel_threshold * static_cast<float>(chan_count)) ? 1 : 0;
  if (!res->detect_enabled) return;
  int nb = 0;
  res->boxcar_length[nb] = 1;
  res->series_length[nb] = ts_count;
  count_signal(ts, ts_count, snr_threshold, &res->variance[nb], &res->threshold[nb],
               &res->signal_count[nb]);
  nb++;
  // inclusive scan, init 0, serial fp32 order (P/algorithm/inclusive_scan.hpp:107-124;
  // the parallel version's order is device dependent)
  std::vector<float> acc(ts_count);
  {
    float a = 0;
    for (size_t i = 0; i < ts_count; i++) {
      a += ts[i];
      acc[i] = a;
    }
  }
  for (size_t b = 2; (b <= max_boxcar_length && b < ts_count) && nb < 32; b *= 2) {
    const size_t n = ts_count - b;
    float* bc = series_out + (size_t)nb * time_count;
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)n; i++) bc[i] = acc[(size_t)i + b] - acc[i];
    res->boxcar_length[nb] = b;
    res->series_length[nb] = n;
    count_signal(bc, n, snr_threshold, &res->variance[nb], &res->threshold[nb],
                 &res->signal_count[nb]);
    nb++;
  }
  res->n_boxcars = nb;
}

// ---------------------------------------------------------------------------
// alternates of the refft path: spectra laid out [time][frequency]
// SK v1 (S/spectrum/rfi_mitigation.hpp:181-275, normalization = false): per frequency column j the sums run over
// the spectra i = 0..M-1 in ascending order, in fp32 (sum_real_t = T, :186).
// ---------------------------------------------------------------------------
void srtb_oracle_sk_v1(float* x_, size_t fft_bins, size_t time_counts, float sk_threshold, float* sk_out,
                       uint8_t* zap) {
  cf* x = reinterpret_cast<cf*>(x_);
  float lo, hi;
  srtb_oracle_sk_thresholds(time_counts, sk_threshold, &lo, &hi);
  std::vector<uint8_t> z(fft_bins);
#pragma omp parallel for schedule(static)
  for (long jj = 0; jj < (long)fft_bins; jj++) {
    const size_t j = (size_t)jj;
    float s2 = 0, s4 = 0;
    for (size_t i = 0; i < time_counts; i++) {
      const float x2 = cnorm(x[i * fft_bins + j]);
      const float x4 = x2 * x2;
      s2 += x2;
      s4 += x4;
    }
    const float sk = static_cast<float>(time_counts) * (s4 / (s2 * s2));
    z[j] = (sk > hi || sk < lo) ? 1 : 0;
    if (sk_out) sk_out[j] = sk;
    if (zap) zap[j] = z[j];
  }
#pragma omp parallel for schedule(static)
  for (long ii = 0; ii < (long)time_counts; ii++)
    for (size_t j = 0; j < fft_bins; j++)
      if (z[j]) x[(size_t)ii * fft_bins + j] = cf{0, 0};
}

// signal_detect_pipe v1 (S/pipeline/signal_detect_pipe.hpp:51-230): x is [batch_size = time][count_per_batch =
// frequency]; SK v1 in place (:66-68), zero_count over the first count_per_batch elements (:74-90), one value per
// spectrum (:93-107; the reference's work-group order is device dependent, ascending order here), mean removal
// (:115-126), count_signal, inclusive scan, boxcars 2, 4, .. (:166-205; nothing is trimmed, lengths n - boxcar).
// series_out rows are batch_size floats apart.
void srtb_oracle_signal_detect_v1(float* x_, size_t count_per_batch, size_t batch_size, float sk_threshold,
                                  float snr_threshold, float channel_threshold, size_t max_boxcar_length,
                                  srtb_oracle_detect_result* res, float* series_out) {
  srtb_oracle_sk_v1(x_, count_per_batch, batch_size, sk_threshold, nullptr, nullptr);
  const cf* x = reinterpret_cast<const cf*>(x_);
  std::memset(res, 0, sizeof(*res));
  uint64_t zero_count = 0;
  for (size_t j = 0; j < count_per_batch; j++)
    if (cnorm(x[j]) == 0) zero_count++;
  res->zero_count = zero_count;
  const size_t n = batch_size;
  res->time_series_count = n;
  float* ts = series_out;
#pragma omp parallel for schedule(static)
  for (long ii = 0; ii < (long)n; ii++) {
    const cf* row = x + (size_t)ii * count_per_batch;
    float s = 0;
    for (size_t j = 0; j < count_per_batch; j++) s += cnorm(row[j]);
    ts[ii] = s;
  }
  const float avg = parallel_pairwise_sum(n, [&](size_t i) { return ts[i]; }) / static_cast<float>(n);
#pragma omp parallel for schedule(static)
  for (long i = 0; i < (long)n; i++) ts[i] -= avg;
  res->detect_enabled =
      (static_cast<float>(zero_count) < channel_threshold * static_cast<float>(count_per_batch)) ? 1 : 0;
  if (!res->detect_enabled) return;
  int nb = 0;
  res->boxcar_length[nb] = 1;
  res->series_length[nb] = n;
  count_signal(ts, n, snr_threshold, &res->variance[nb], &res->threshold[nb], &res->signal_count[nb]);
  nb++;
  std::vector<float> acc(n);
  {
    float a = 0;
    for (size_t i = 0; i < n; i++) {
      a += ts[i];
      acc[i] = a;
    }
  }
  for (size_t b = 2; (b <= max_boxcar_length && b < n) && nb < 32; b *= 2) {
    const size_t m = n - b;
    float* bc = series_out + (size_t)nb * n;
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)m; i++) bc[i] = acc[(size_t)i + b] - acc[i];
    res->boxcar_length[nb] = b;
    res->series_length[nb] = m;
    count_signal(bc, m, snr_threshold, &res->variance[nb], &res->threshold[nb], &res->signal_count[nb]);
    nb++;
  }
  res->n_boxcars = nb;
}

// ---------------------------------------------------------------------------
// whole chain on one stream ("simple" format) — used as the CPU baseline.
// work = caller buffer of N+2 floats. Returns 0 on success.
// fft_kind: 0 = restated naive radix-2 (what the reference runs without FFTW,
//           S/fft/fft.hpp:22-26,143).
// ---------------------------------------------------------------------------
struct srtb_oracle_chain_config {
  uint64_t baseband_input_count;  // N (samples)
  int32_t baseband_input_bits;
  int32_t window;
  float baseband_freq_low, baseband_bandwidth, baseband_sample_rate, dm;
  int32_t baseband_reserve_sample;
  float rfi_average_threshold, rfi_sk_threshold;
  uint64_t spectrum_channel_count;
  float snr_threshold, channel_threshold;
  uint64_t max_boxcar_length;
  const float* rfi_pairs;
  uint64_t n_rfi_pairs;
};

int srtb_oracle_chain(const void* baseband, const srtb_oracle_chain_config* cfg, float* work,
                      srtb_oracle_detect_result* res, float* series_out, double* stage_seconds) {
  auto now = []() {
#if defined(_OPENMP)
    return omp_get_wtime();
#else
    return 0.0;
#endif
  };
  const size_t N = cfg->baseband_input_count;
  double t0 = now();
  if (srtb_oracle_unpack(baseband, N, cfg->baseband_input_bits, cfg->window, work) != 0) return -1;
  double t1 = now();
  srtb_oracle_fft_r2c(work, N);
  double t2 = now();
  const size_t Nc = N / 2;
  srtb_oracle_rfi_s1_average(work, Nc, cfg->rfi_average_threshold, cfg->spectrum_channel_count,
                             nullptr, nullptr);
  srtb_oracle_rfi_manual(work, Nc, cfg->baseband_freq_low, cfg->baseband_bandwidth, cfg->rfi_pairs,
                         cfg->n_rfi_pairs);
  double t3 = now();
  const float df = cfg->baseband_bandwidth / static_cast<float>(Nc);  // dedisperse_pipe.hpp:34
  const float f_min = cfg->baseband_freq_low, f_c = f_min + cfg->baseband_bandwidth;
  srtb_oracle_dedisperse(work, Nc, f_min, f_c, df, cfg->dm);
  double t4 = now();
  const size_t batch = std::min((size_t)cfg->spectrum_channel_count, Nc);  // fft_pipe.hpp:318-320
  const size_t L = Nc / batch;
  srtb_oracle_watfft(work, L, batch);
  double t5 = now();
  srtb_oracle_rfi_s2(work, L, batch, cfg->rfi_sk_threshold, nullptr, nullptr);
  double t6 = now();
  const size_t reserved =
      srtb_oracle_nsamps_reserved(N, cfg->spectrum_channel_count, cfg->baseband_freq_low,
                                  cfg->baseband_bandwidth, cfg->baseband_sample_rate, cfg->dm,
                                  cfg->baseband_reserve_sample) /
      batch;
  srtb_oracle_signal_detect(work, L, batch, reserved, cfg->snr_threshold, cfg->channel_threshold,
                            cfg->max_boxcar_length, res, series_out);
  double t7 = now();
  if (stage_seconds) {
    stage_seconds[0] = t1 - t0;
    stage_seconds[1] = t2 - t1;
    stage_seconds[2] = t3 - t2;
    stage_seconds[3] = t4 - t3;
    stage_seconds[4] = t5 - t4;
    stage_seconds[5] = t6 - t5;
    stage_seconds[6] = t7 - t6;
  }
  return 0;
}

void srtb_oracle_set_threads(int n) {
#if defined(_OPENMP)
  if (n > 0) omp_set_num_threads(n);
#else
  (void)n;
#endif
}

// count_signal of one series (signal_detect.hpp:32-72): elements above snr * sqrt(mean(v^2))
uint64_t srtb_oracle_count_signal(const float* v, size_t n, float snr) {
  float var = 0, thr = 0;
  uint64_t cnt = 0;
  count_signal(v, n, snr, &var, &thr, &cnt);
  return cnt;
}

int srtb_oracle_num_threads(void) {
#if defined(_OPENMP)
  return omp_get_max_threads();
#else
  return 1;
#endif
}

}  // extern "C"
