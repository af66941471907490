// ops_kernels.cuh — the non-FFT kernels of the path, hand-written for sm_90a.
// All are HBM-bound streaming kernels: 16-byte vector accesses, fully coalesced,
// grid sized as a multiple of the SM count, reductions by warp shuffles.
// Reference operators are cited per kernel (S/ = userspace/include/srtb/).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace srtb_b200 {

// ------------------------------------------------------------------------------
// FFT window (S/fft/fft_window.hpp:27-50,112-123): w(i) = sum_k (-1)^k a_k cos(2 pi k x),
// x = float(i) / float(n - 1), the cosine evaluated in double as the reference's
// `2 * M_PI * k * x` expression is. window 0 = rectangle (identity, the default).
// ------------------------------------------------------------------------------
__device__ __forceinline__ float window_value(int window, size_t i, float n_minus_1) {
  if (window == 0) return 1.0f;
  const float a0 = (window == 1) ? 0.5f : (float)(25.0 / 46.0);
  const float a1 = (window == 1) ? 0.5f : (float)(21.0 / 46.0);
  const float x = (float)i / n_minus_1;
  float ret = 0.0f;
  ret = (float)((double)ret + (double)a0 * cos(2.0 * 3.14159265358979323846 * 0.0 * (double)x));
  ret = (float)((double)ret + (double)(-a1) * cos(2.0 * 3.14159265358979323846 * 1.0 * (double)x));
  return ret;
}

// ------------------------------------------------------------------------------
// K1 unpack "simple" (S/unpack.hpp:43-156,171-197). unpack_src<> (8 samples at a time) serves
// the de-interleaving kernels; unpack_quad<> (one float4) serves the simple kernel.
// ------------------------------------------------------------------------------
template <int BITS>
struct unpack_src {};  // loads the bytes of 8 consecutive samples starting at sample 8*g

template <>
struct unpack_src<1> {
  __device__ static void get(const void* in, size_t g, float (&o)[8]) {
    const unsigned v = static_cast<const uint8_t*>(in)[g];
#pragma unroll
    for (int i = 0; i < 8; i++) o[i] = (float)((v >> (7 - i)) & 1u);
  }
};
template <>
struct unpack_src<2> {
  __device__ static void get(const void* in, size_t g, float (&o)[8]) {
    const unsigned v = static_cast<const uint16_t*>(in)[g];  // little endian: byte 0 = low
#pragma unroll
    for (int i = 0; i < 4; i++) o[i] = (float)(((v & 0xffu) >> (6 - 2 * i)) & 3u);
#pragma unroll
    for (int i = 0; i < 4; i++) o[4 + i] = (float)(((v >> 8) >> (6 - 2 * i)) & 3u);
  }
};
template <>
struct unpack_src<4> {
  __device__ static void get(const void* in, size_t g, float (&o)[8]) {
    const unsigned v = static_cast<const uint32_t*>(in)[g];
#pragma unroll
    for (int b = 0; b < 4; b++) {
      const unsigned byte = (v >> (8 * b)) & 0xffu;
      o[2 * b] = (float)(byte >> 4);
      o[2 * b + 1] = (float)(byte & 0xfu);
    }
  }
};
template <>
struct unpack_src<8> {
  __device__ static void get(const void* in, size_t g, float (&o)[8]) {
    const uint2 v = static_cast<const uint2*>(in)[g];
#pragma unroll
    for (int b = 0; b < 4; b++) {
      o[b] = (float)((v.x >> (8 * b)) & 0xffu);
      o[4 + b] = (float)((v.y >> (8 * b)) & 0xffu);
    }
  }
};
template <>
struct unpack_src<-8> {
  __device__ static void get(const void* in, size_t g, float (&o)[8]) {
    const uint2 v = static_cast<const uint2*>(in)[g];
#pragma unroll
    for (int b = 0; b < 4; b++) {
      o[b] = (float)(int)(int8_t)((v.x >> (8 * b)) & 0xffu);
      o[4 + b] = (float)(int)(int8_t)((v.y >> (8 * b)) & 0xffu);
    }
  }
};
template <>
struct unpack_src<16> {
  __device__ static void get(const void* in, size_t g, float (&o)[8]) {
    const uint4 v = static_cast<const uint4*>(in)[g];
    const unsigned w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int b = 0; b < 4; b++) {
      o[2 * b] = (float)(w[b] & 0xffffu);
      o[2 * b + 1] = (float)(w[b] >> 16);
    }
  }
};
template <>
struct unpack_src<-16> {
  __device__ static void get(const void* in, size_t g, float (&o)[8]) {
    const uint4 v = static_cast<const uint4*>(in)[g];
    const unsigned w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int b = 0; b < 4; b++) {
      o[2 * b] = (float)(int)(int16_t)(w[b] & 0xffffu);
      o[2 * b + 1] = (float)(int)(int16_t)(w[b] >> 16);
    }
  }
};
template <>
struct unpack_src<32> {
  __device__ static void get(const void* in, size_t g, float (&o)[8]) {
    const float4 a = static_cast<const float4*>(in)[2 * g], b = static_cast<const float4*>(in)[2 * g + 1];
    o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w;
    o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
  }
};
template <>
struct unpack_src<64> {
  __device__ static void get(const void* in, size_t g, float (&o)[8]) {
    const double2* p = static_cast<const double2*>(in) + 4 * g;
#pragma unroll
    for (int b = 0; b < 4; b++) {
      const double2 d = p[b];
      o[2 * b] = (float)d.x;
      o[2 * b + 1] = (float)d.y;
    }
  }
};

// scalar element access for tails and unaligned inputs
template <int BITS>
__device__ __forceinline__ float unpack_one(const void* in, size_t i) {
  if (BITS == 1 || BITS == 2 || BITS == 4) {
    constexpr int B = (BITS > 0 && BITS < 8) ? BITS : 1;
    constexpr int CNT = 8 / B;
    const unsigned v = static_cast<const uint8_t*>(in)[i / CNT];
    const int j = (int)(i % CNT);
    return (float)((v >> ((CNT - 1 - j) * B)) & ((1u << B) - 1u));
  }
  if (BITS == 8) return (float)static_cast<const uint8_t*>(in)[i];
  if (BITS == -8) return (float)static_cast<const int8_t*>(in)[i];
  if (BITS == 16) return (float)static_cast<const uint16_t*>(in)[i];
  if (BITS == -16) return (float)static_cast<const int16_t*>(in)[i];
  if (BITS == 32) return static_cast<const float*>(in)[i];
  return (float)static_cast<const double*>(in)[i];
}

// one float4 of output (samples 4q .. 4q+3) from the 4*|BITS| input bits it needs
template <int BITS>
__device__ __forceinline__ float4 unpack_quad(const void* __restrict__ in, size_t q) {
  if (BITS == 1) {
    const unsigned v = static_cast<const uint8_t*>(in)[q >> 1];
    const unsigned nib = (q & 1) ? (v & 0xfu) : (v >> 4);
    return make_float4((float)((nib >> 3) & 1u), (float)((nib >> 2) & 1u), (float)((nib >> 1) & 1u), (float)(nib & 1u));
  } else if (BITS == 2) {
    const unsigned v = static_cast<const uint8_t*>(in)[q];
    return make_float4((float)(v >> 6), (float)((v >> 4) & 3u), (float)((v >> 2) & 3u), (float)(v & 3u));
  } else if (BITS == 4) {
    const unsigned v = static_cast<const uint16_t*>(in)[q];  // little endian: byte 0 first
    return make_float4((float)((v >> 4) & 0xfu), (float)(v & 0xfu), (float)(v >> 12), (float)((v >> 8) & 0xfu));
  } else if (BITS == 8) {
    const unsigned v = static_cast<const uint32_t*>(in)[q];
    return make_float4((float)(v & 0xffu), (float)((v >> 8) & 0xffu), (float)((v >> 16) & 0xffu), (float)(v >> 24));
  } else if (BITS == -8) {
    const unsigned v = static_cast<const uint32_t*>(in)[q];
    return make_float4((float)(int)(int8_t)(v & 0xffu), (float)(int)(int8_t)((v >> 8) & 0xffu),
                       (float)(int)(int8_t)((v >> 16) & 0xffu), (float)(int)(int8_t)(v >> 24));
  } else if (BITS == 16) {
    const uint2 v = static_cast<const uint2*>(in)[q];
    return make_float4((float)(v.x & 0xffffu), (float)(v.x >> 16), (float)(v.y & 0xffffu), (float)(v.y >> 16));
  } else if (BITS == -16) {
    const uint2 v = static_cast<const uint2*>(in)[q];
    return make_float4((float)(int)(int16_t)(v.x & 0xffffu), (float)(int)(int16_t)(v.x >> 16),
                       (float)(int)(int16_t)(v.y & 0xffffu), (float)(int)(int16_t)(v.y >> 16));
  } else if (BITS == 32) {
    return static_cast<const float4*>(in)[q];
  } else {
    const double2 a = static_cast<const double2*>(in)[2 * q], b2 = static_cast<const double2*>(in)[2 * q + 1];
    return make_float4((float)a.x, (float)a.y, (float)b2.x, (float)b2.y);
  }
}

// K1: every warp-level access is contiguous (32 lanes x 16 B stores = 512 B; loads 32 x |BITS|/2 B);
// four independent quads per thread per iteration keep 4 loads + 4 stores in flight.
template <int BITS, bool WIN>
__global__ void __launch_bounds__(256) unpack_simple_kernel(const void* __restrict__ in,
                                                            float* __restrict__ out, size_t n,
                                                            int window) {
  constexpr int K = 4;
  const size_t quads = n / 4;
  const float nm1 = (float)(n - 1);
  const size_t stride = (size_t)gridDim.x * blockDim.x * K;
  float4* __restrict__ dst = reinterpret_cast<float4*>(out);
  for (size_t q0 = (size_t)blockIdx.x * blockDim.x * K + threadIdx.x; q0 < quads; q0 += stride) {
    float4 v[K];
#pragma unroll
    for (int j = 0; j < K; j++) {
      const size_t q = q0 + (size_t)j * blockDim.x;
      if (q < quads) v[j] = unpack_quad<BITS>(in, q);
    }
#pragma unroll
    for (int j = 0; j < K; j++) {
      const size_t q = q0 + (size_t)j * blockDim.x;
      if (q < quads) {
        if (WIN) {
          v[j].x *= window_value(window, 4 * q, nm1);
          v[j].y *= window_value(window, 4 * q + 1, nm1);
          v[j].z *= window_value(window, 4 * q + 2, nm1);
          v[j].w *= window_value(window, 4 * q + 3, nm1);
        }
        dst[q] = v[j];
      }
    }
  }
  // tail (n % 4 samples) by the first threads of block 0
  if (blockIdx.x == 0) {
    const size_t i = quads * 4 + threadIdx.x;
    if (threadIdx.x < 4 && i < n) {
      float v = unpack_one<BITS>(in, i);
      if (WIN) v *= window_value(window, i, nm1);
      out[i] = v;
    }
  }
}

// scalar fallback for inputs whose base pointer is not 16-byte aligned
template <int BITS>
__global__ void __launch_bounds__(256) unpack_simple_scalar_kernel(const void* __restrict__ in,
                                                                   float* __restrict__ out, size_t n,
                                                                   int window) {
  const float nm1 = (float)(n - 1);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    out[i] = unpack_one<BITS>(in, i) * window_value(window, i, nm1);
}

// K2 "1 2 1 2" de-interleave (S/unpack.hpp:221-244): thread writes 4 samples per stream
template <int BITS>
__global__ void __launch_bounds__(256) unpack_interleaved2_kernel(const void* __restrict__ in,
                                                                  float* __restrict__ o1,
                                                                  float* __restrict__ o2, size_t n,
                                                                  int window) {
  const float nm1 = (float)(n - 1);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t groups = n / 4;
  for (size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += stride) {
    float o[8];
    unpack_src<BITS>::get(in, g, o);  // 8 interleaved samples = 4 per stream
    float a[4] = {o[0], o[2], o[4], o[6]}, b[4] = {o[1], o[3], o[5], o[7]};
    if (window != 0) {
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const float w = window_value(window, 4 * g + i, nm1);
        a[i] *= w;
        b[i] *= w;
      }
    }
    reinterpret_cast<float4*>(o1)[g] = make_float4(a[0], a[1], a[2], a[3]);
    reinterpret_cast<float4*>(o2)[g] = make_float4(b[0], b[1], b[2], b[3]);
  }
  if (blockIdx.x == 0 && threadIdx.x < 4) {
    const size_t i = groups * 4 + threadIdx.x;
    if (i < n) {
      const float w = window_value(window, i, nm1);
      o1[i] = unpack_one<BITS>(in, 2 * i) * w;
      o2[i] = unpack_one<BITS>(in, 2 * i + 1) * w;
    }
  }
}

// K3 naocpsr_snap1 "1 1 2 2" int8 (S/unpack.hpp:255-283)
__global__ void __launch_bounds__(256) unpack_snap1_kernel(const void* __restrict__ in,
                                                           float* __restrict__ o1,
                                                           float* __restrict__ o2, size_t n,
                                                           int window) {
  const float nm1 = (float)(n - 1);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t groups = n / 4;  // 4 samples per stream = 8 input bytes
  for (size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += stride) {
    float o[8];
    unpack_src<-8>::get(in, g, o);  // a0 a1 b0 b1 a2 a3 b2 b3
    float a[4] = {o[0], o[1], o[4], o[5]}, b[4] = {o[2], o[3], o[6], o[7]};
    if (window != 0) {
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const float w = window_value(window, 4 * g + i, nm1);
        a[i] *= w;
        b[i] *= w;
      }
    }
    reinterpret_cast<float4*>(o1)[g] = make_float4(a[0], a[1], a[2], a[3]);
    reinterpret_cast<float4*>(o2)[g] = make_float4(b[0], b[1], b[2], b[3]);
  }
  // tail: the reference launches n/2 work items of 2 samples per stream (:280-282)
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const int8_t* p = static_cast<const int8_t*>(in);
    for (size_t x = groups * 2; x < n / 2; x++) {
      o1[2 * x] = (float)p[4 * x] * window_value(window, 2 * x, nm1);
      o1[2 * x + 1] = (float)p[4 * x + 1] * window_value(window, 2 * x + 1, nm1);
      o2[2 * x] = (float)p[4 * x + 2] * window_value(window, 2 * x, nm1);
      o2[2 * x + 1] = (float)p[4 * x + 3] * window_value(window, 2 * x + 1, nm1);
    }
  }
}

// K4 gznupsr_a1 (S/unpack.hpp:293-403): 4-sample words round-robin to S streams.
// S = 4 applies float(int(int8) ^ 0x80) (:315-316); S = 2 does not (:356-357).
template <int S>
__global__ void __launch_bounds__(256) unpack_gznupsr_kernel(const void* __restrict__ in,
                                                             float* __restrict__ o0,
                                                             float* __restrict__ o1,
                                                             float* __restrict__ o2,
                                                             float* __restrict__ o3, size_t n,
                                                             int window) {
  const float nm1 = (float)(n - 1);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t words = n / 4;
  float* outs[4] = {o0, o1, o2, o3};
  for (size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x; x < words; x += stride) {
    unsigned w[4];
    if (S == 4) {
      const uint4 v = static_cast<const uint4*>(in)[x];
      w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
    } else {
      const uint2 v = static_cast<const uint2*>(in)[x];
      w[0] = v.x; w[1] = v.y; w[2] = 0; w[3] = 0;
    }
    float wv[4] = {1.f, 1.f, 1.f, 1.f};
    if (window != 0) {
#pragma unroll
      for (int j = 0; j < 4; j++) wv[j] = window_value(window, 4 * x + j, nm1);
    }
#pragma unroll
    for (int i = 0; i < S; i++) {
      float f[4];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int s = (int)(int8_t)((w[i] >> (8 * j)) & 0xffu);
        f[j] = (S == 4) ? (float)(s ^ 0x80) : (float)s;
        f[j] *= wv[j];
      }
      reinterpret_cast<float4*>(outs[i])[x] = make_float4(f[0], f[1], f[2], f[3]);
    }
  }
}

// ------------------------------------------------------------------------------
// K8 R2C split post-process (S/fft/naive_fft.hpp:229-260), in place on M + 1 bins:
// H = FFT_M(x_even + i x_odd);  F = (H_k + conj H_{M-k})/2, G = -i (H_k - conj H_{M-k})/2,
// X_k = F + G w,  X_{M-k} = conj(F - G w),  w = e^{-i pi k / M};  k = 0 also writes X_M.
// ------------------------------------------------------------------------------
__device__ __forceinline__ float2 r2c_twiddle(size_t k, size_t M) {
  // e^{-i pi k / M}; k/M is exact in fp32 while k < 2^24, otherwise split k = kh*2^12 + kl
  float s, c;
  if (M <= ((size_t)1 << 25)) {
    sincospif(-(float)k / (float)M, &s, &c);
    return make_float2(c, s);
  }
  const size_t kh = k >> 12, kl = k & 4095;
  float s1, c1, s2, c2;
  sincospif(-(float)kh / (float)(M >> 12), &s1, &c1);
  sincospif(-(float)kl / (float)M, &s2, &c2);
  return make_float2(c1 * c2 - s1 * s2, c1 * s2 + s1 * c2);
}

// ------------------------------------------------------------------------------
// reductions
// ------------------------------------------------------------------------------
__host__ __device__ __forceinline__ bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// block-wide sum; result valid in thread 0. sm must hold 32 values.
template <typename T>
__device__ __forceinline__ T block_sum(T v, T* sm) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) sm[wid] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  T r = (threadIdx.x < nw) ? sm[threadIdx.x] : T(0);
  if (wid == 0) r = warp_sum(r);
  return r;
}

// SUM = true additionally produces the mean of |X_k|^2 over k < M (the s1 statistic, K9) while the
// bins are in registers: per-CTA fp64 partials + last-CTA ticket, exactly as power_sum_kernel.
template <bool SUM>
__global__ void __launch_bounds__(256) r2c_post_kernel(float2* __restrict__ H, size_t M,
                                                       double* __restrict__ partial,
                                                       unsigned* __restrict__ ticket,
                                                       float* __restrict__ mean_out) {
  __shared__ double sm[32];
  __shared__ bool last;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  float acc = 0.f;
  auto split = [&](size_t k, float2 hk, float2 hm) {
    const float2 F = make_float2(0.5f * (hk.x + hm.x), 0.5f * (hk.y - hm.y));
    // d = hk - conj(hm) = (hk.x - hm.x, hk.y + hm.y);  G = -i/2 * d = (d.y/2, -d.x/2)
    const float2 G = make_float2(0.5f * (hk.y + hm.y), -0.5f * (hk.x - hm.x));
    const float2 w = r2c_twiddle(k, M);
    const float2 gw = make_float2(G.x * w.x - G.y * w.y, G.x * w.y + G.y * w.x);
    const float2 xk = make_float2(F.x + gw.x, F.y + gw.y);
    const float2 xm = make_float2(F.x - gw.x, -(F.y - gw.y));
    H[k] = xk;
    H[M - k] = xm;  // k == M/2 writes the same bin twice; the reference keeps this one (:257-258)
    if (SUM) {
      // bins 0 .. M-1 count (the Nyquist bin M is dropped by the pipe); bin M/2 counted once
      const float wm = (k == 0 || 2 * k == M) ? 0.f : 1.f;
      acc += (xk.x * xk.x + xk.y * xk.y) + wm * (xm.x * xm.x + xm.y * xm.y);
    }
  };
  size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; k + stride <= M / 2; k += 2 * stride) {   // two independent pairs: four loads in flight
    const size_t k2 = k + stride;
    const float2 a0 = H[k], a1 = (k == 0) ? a0 : H[M - k];
    const float2 b0 = H[k2], b1 = H[M - k2];
    split(k, a0, a1);
    split(k2, b0, b1);
  }
  if (k <= M / 2) {
    const float2 a0 = H[k], a1 = (k == 0) ? a0 : H[M - k];
    split(k, a0, a1);
  }
  if (SUM) {
    const double s = block_sum<double>((double)acc, sm);
    if (threadIdx.x == 0) {
      partial[blockIdx.x] = s;
      __threadfence();
      last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
      if (last) __threadfence();  // one acquiring fence (a fence per warp serialises: ~1 us each)
    }
    __syncthreads();
    if (last) {
      double a = 0.0;
      for (unsigned i = threadIdx.x; i < gridDim.x; i += blockDim.x) a += partial[i];
      a = block_sum<double>(a, sm);
      if (threadIdx.x == 0) {
        *mean_out = (float)a / (float)M;
        *ticket = 0;
      }
    }
  }
}

// K9 mean of |X|^2 (S/algorithm/map_reduce.hpp:84-91 over rfi_mitigation_pipe.hpp:53-60).
// fp32 per-thread partials, fp64 combine, deterministic: per-CTA partials are summed in
// index order by the last CTA to finish. mean = float(sum) / float(count).
// A spectrum that is only 8-byte aligned (a complex64 view starting at an odd element) is read one element at a time.
__global__ void __launch_bounds__(256) power_sum_kernel(const float2* __restrict__ x, size_t count,
                                                        double* __restrict__ partial,
                                                        unsigned* __restrict__ ticket,
                                                        float* __restrict__ mean_out) {
  __shared__ double sm[32];
  __shared__ bool last;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t pairs = count / 2;
  float acc0 = 0.f, acc1 = 0.f;
  const float4* x4 = reinterpret_cast<const float4*>(x);
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (!aligned16(x)) {
    for (size_t j = i; j < count; j += stride) {
      const float2 v = x[j];
      acc0 += v.x * v.x + v.y * v.y;
    }
    i = pairs;  // skip the vector loops and the odd tail below
  }
  for (; i + 3 * stride < pairs; i += 4 * stride) {   // four loads in flight per thread
    const float4 a = x4[i], b = x4[i + stride], c = x4[i + 2 * stride], d = x4[i + 3 * stride];
    acc0 += (a.x * a.x + a.y * a.y) + (b.x * b.x + b.y * b.y);
    acc1 += (a.z * a.z + a.w * a.w) + (b.z * b.z + b.w * b.w);
    acc0 += (c.x * c.x + c.y * c.y) + (d.x * d.x + d.y * d.y);
    acc1 += (c.z * c.z + c.w * c.w) + (d.z * d.z + d.w * d.w);
  }
  for (; i < pairs; i += stride) {
    const float4 v = x4[i];
    acc0 += v.x * v.x + v.y * v.y;
    acc1 += v.z * v.z + v.w * v.w;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0 && (count & 1) && aligned16(x)) {
    const float2 v = x[count - 1];
    acc0 += v.x * v.x + v.y * v.y;
  }
  const double s = block_sum<double>((double)acc0 + (double)acc1, sm);
  if (threadIdx.x == 0) {
    partial[blockIdx.x] = s;
    __threadfence();
    const unsigned t = atomicAdd(ticket, 1u);
    last = (t == gridDim.x - 1);
    if (last) __threadfence();  // one acquiring fence (a fence per warp serialises: ~1 us each)
  }
  __syncthreads();
  if (last) {
    double a = 0.0;
    for (unsigned i = threadIdx.x; i < gridDim.x; i += blockDim.x) a += partial[i];
    a = block_sum<double>(a, sm);
    if (threadIdx.x == 0) {
      *mean_out = (float)a / (float)count;
      *ticket = 0;
    }
  }
}

// K10 zap + normalise (S/pipeline/rfi_mitigation_pipe.hpp:66-79)
__global__ void __launch_bounds__(256) rfi_s1_apply_kernel(float2* __restrict__ x, size_t count,
                                                           const float* __restrict__ mean,
                                                           float threshold, float coef) {
  const float limit = threshold * (*mean);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  if (!aligned16(x)) {  // 8-byte aligned spectrum: one element per load
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) {
      float2 v = x[i];
      if (v.x * v.x + v.y * v.y > limit) v = make_float2(0.f, 0.f);
      else { v.x *= coef; v.y *= coef; }
      x[i] = v;
    }
    return;
  }
  const size_t pairs = count / 2;
  float4* x4 = reinterpret_cast<float4*>(x);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < pairs; i += stride) {
    float4 v = x4[i];
    const float p0 = v.x * v.x + v.y * v.y, p1 = v.z * v.z + v.w * v.w;
    if (p0 > limit) { v.x = 0.f; v.y = 0.f; } else { v.x *= coef; v.y *= coef; }
    if (p1 > limit) { v.z = 0.f; v.w = 0.f; } else { v.z *= coef; v.w *= coef; }
    x4[i] = v;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0 && (count & 1)) {
    float2 v = x[count - 1];
    if (v.x * v.x + v.y * v.y > limit) v = make_float2(0.f, 0.f);
    else { v.x *= coef; v.y *= coef; }
    x[count - 1] = v;
  }
}

// K11 manual zap (S/spectrum/rfi_mitigation.hpp:137-143): blockIdx.y = range
// logp != 0: the spectrum is channel-blocked (r2c_rows_split_kernel): bin k = k1 + 2^logp k2 at
// (k2 >> 3) 2^logq + 8 k1 + (k2 & 7), channels of 2^logq = 8 2^logp bins
struct bin_ranges {
  unsigned long long lo[16], hi[16];
  unsigned logp, logq;
};
__global__ void __launch_bounds__(256) rfi_zero_ranges_kernel(float2* __restrict__ x, bin_ranges r) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t lo = r.lo[blockIdx.y], hi = r.hi[blockIdx.y];
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t pmask = ((size_t)1 << r.logp) - 1;
  for (size_t i = lo + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i <= hi; i += stride) {
    const size_t k1 = i & pmask, k2 = i >> r.logp;
    x[r.logp ? ((k2 >> 3) << r.logq) + 8 * k1 + (k2 & 7) : i] = make_float2(0.f, 0.f);
  }
}

// ------------------------------------------------------------------------------
// K12 chirp multiply (S/coherent_dedispersion.hpp:133-150 phase_factor_v3, :228-236).
// f = f_min + df*i in fp64 (f32 inputs promoted), k = (D*1e6*dm)/f * ((f-f_c)/f_c)^2,
// phi = -2 pi frac(k); the sincos is taken as sincospi(-2 frac) in fp32.
// ------------------------------------------------------------------------------
// chirp_factor() lives in fft_engine.cuh (shared with the fused waterfall kernel)

// S1 = true fuses K10 (zap + normalise, rfi_mitigation_pipe.hpp:66-79) in front of the chirp: used by
// srtb_b200_process_block, where the s1 and dedisperse pipes run back to back on one stream.
// `in` may equal `out` (in place, the pipe's contract) or differ (DM sweep: the spectrum is kept).
template <bool S1>
__global__ void __launch_bounds__(256) dedisperse_kernel(const float2* in, float2* x, size_t count,
                                                         double f_min, double df, double f_c,
                                                         double ddm, const float* __restrict__ mean,
                                                         float threshold, float coef) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t pairs = count / 2;
  const double inv_fc = 1.0 / f_c;
  const float limit = S1 ? threshold * (*mean) : 0.f;
  if (!aligned16(in) || !aligned16(x)) {  // 8-byte aligned spectra: one element per load
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) {
      float2 v = in[i];
      if (S1) {
        if (v.x * v.x + v.y * v.y > limit) v = make_float2(0.f, 0.f);
        else { v.x *= coef; v.y *= coef; }
      }
      const float2 w = chirp_factor(f_min, df, inv_fc, f_c, ddm, (unsigned)i);
      x[i] = make_float2(v.x * w.x - v.y * w.y, v.x * w.y + v.y * w.x);
    }
    return;
  }
  float4* x4 = reinterpret_cast<float4*>(x);
  const float4* in4 = reinterpret_cast<const float4*>(in);
  auto one = [&](float4 v, size_t i) {
    if (S1) {
      const float p0 = v.x * v.x + v.y * v.y, p1 = v.z * v.z + v.w * v.w;
      if (p0 > limit) { v.x = 0.f; v.y = 0.f; } else { v.x *= coef; v.y *= coef; }
      if (p1 > limit) { v.z = 0.f; v.w = 0.f; } else { v.z *= coef; v.w *= coef; }
    }
    const float2 w0 = chirp_factor(f_min, df, inv_fc, f_c, ddm, (unsigned)(2 * i));
    const float2 w1 = chirp_factor(f_min, df, inv_fc, f_c, ddm, (unsigned)(2 * i + 1));
    x4[i] = make_float4(v.x * w0.x - v.y * w0.y, v.x * w0.y + v.y * w0.x,
                        v.z * w1.x - v.w * w1.y, v.z * w1.y + v.w * w1.x);
  };
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + stride < pairs; i += 2 * stride) {  // two independent 16-byte loads in flight per thread
    const float4 a = in4[i], b = in4[i + stride];
    one(a, i);
    one(b, i + stride);
  }
  if (i < pairs) one(in4[i], i);
  if (blockIdx.x == 0 && threadIdx.x == 0 && (count & 1)) {
    float2 v = in[count - 1];
    if (S1) {
      if (v.x * v.x + v.y * v.y > limit) v = make_float2(0.f, 0.f);
      else { v.x *= coef; v.y *= coef; }
    }
    const float2 w = chirp_factor(f_min, df, inv_fc, f_c, ddm, (unsigned)(count - 1));
    x[count - 1] = make_float2(v.x * w.x - v.y * w.y, v.x * w.y + v.y * w.x);
  }
}

// ------------------------------------------------------------------------------
// K14 + K15 spectral kurtosis (S/spectrum/rfi_mitigation.hpp:292-341; sums by
// S/algorithm/multi_reduce.hpp:115-155). One CTA per channel row: s2, s4, decide, zero.
// ------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) sk_kernel(float2* __restrict__ x, size_t time_count,
                                                 float thr_lo, float thr_hi,
                                                 float* __restrict__ sk_out) {
  __shared__ float sm[32];
  __shared__ int zap;
  float2* row = x + (size_t)blockIdx.x * time_count;
  float s2 = 0.f, s4 = 0.f;
  const size_t pairs = time_count / 2;
  const float4* r4 = reinterpret_cast<const float4*>(row);
  const bool vec = aligned16(row);
  if (vec) {
    size_t i = threadIdx.x;
    const size_t bd = blockDim.x;
    for (; i + 3 * bd < pairs; i += 4 * bd) {   // four loads in flight per thread
      const float4 a = r4[i], b = r4[i + bd], c = r4[i + 2 * bd], d = r4[i + 3 * bd];
      const float pa0 = a.x * a.x + a.y * a.y, pa1 = a.z * a.z + a.w * a.w;
      const float pb0 = b.x * b.x + b.y * b.y, pb1 = b.z * b.z + b.w * b.w;
      const float pc0 = c.x * c.x + c.y * c.y, pc1 = c.z * c.z + c.w * c.w;
      const float pd0 = d.x * d.x + d.y * d.y, pd1 = d.z * d.z + d.w * d.w;
      s2 += (pa0 + pa1) + (pb0 + pb1) + (pc0 + pc1) + (pd0 + pd1);
      s4 += (pa0 * pa0 + pa1 * pa1) + (pb0 * pb0 + pb1 * pb1) + (pc0 * pc0 + pc1 * pc1) + (pd0 * pd0 + pd1 * pd1);
    }
    for (; i < pairs; i += bd) {
      const float4 v = r4[i];
      const float p0 = v.x * v.x + v.y * v.y, p1 = v.z * v.z + v.w * v.w;
      s2 += p0 + p1;
      s4 += p0 * p0 + p1 * p1;
    }
    if (threadIdx.x == 0 && (time_count & 1)) {
      const float2 v = row[time_count - 1];
      const float p = v.x * v.x + v.y * v.y;
      s2 += p;
      s4 += p * p;
    }
  } else {
    for (size_t i = threadIdx.x; i < time_count; i += blockDim.x) {
      const float2 v = row[i];
      const float p = v.x * v.x + v.y * v.y;
      s2 += p;
      s4 += p * p;
    }
  }
  const float t2 = block_sum<float>(s2, sm);
  const float t4 = block_sum<float>(s4, sm);
  if (threadIdx.x == 0) {
    const float sk = (float)time_count * (t4 / (t2 * t2));
    zap = (sk > thr_hi || sk < thr_lo) ? 1 : 0;  // NaN compares false: row left as is
    if (sk_out) sk_out[blockIdx.x] = sk;
  }
  __syncthreads();
  if (zap) {
    for (size_t i = threadIdx.x; i < time_count; i += blockDim.x) row[i] = make_float2(0.f, 0.f);
  }
}

// ------------------------------------------------------------------------------
// signal detect (S/pipeline/signal_detect_pipe.hpp:252-442, S/signal_detect.hpp:32-72)
// ------------------------------------------------------------------------------
struct detect_dev_result {
  unsigned long long zero_count;
  unsigned long long time_series_count;
  int detect_enabled;
  int n_boxcars;
  unsigned long long boxcar_length[32];
  unsigned long long series_length[32];
  unsigned long long signal_count[32];
  float variance[32];
  float threshold[32];
};
// srtb_b200_peak: per boxcar, the largest series value over sqrt(variance) and the first index that reaches it
struct detect_dev_peak {
  float snr[32];
  unsigned long long peak_index[32];
};

// K14 for long rows (process_block, rows above 2^14): the last waterfall sweep left per-tile (sum |y|^2, sum |y|^4);
// one thread per channel row folds its tiles in index order and decides (rfi_mitigation.hpp:292-341; NaN -> keep)
__global__ void __launch_bounds__(256) sk_decide_kernel(const float2* __restrict__ tile_stats, unsigned tiles_per_row,
                                                        size_t chan_count, float m_count, float thr_lo, float thr_hi,
                                                        unsigned char* __restrict__ zap) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= chan_count) return;
  float s2 = 0.f, s4 = 0.f;
  for (unsigned t = 0; t < tiles_per_row; t++) {
    const float2 v = tile_stats[c * tiles_per_row + t];
    s2 += v.x;
    s4 += v.y;
  }
  const float sk = m_count * (s4 / (s2 * s2));
  zap[c] = (sk > thr_hi || sk < thr_lo) ? 1 : 0;
}

// K17 stage 1: partial column sums over a chunk of channels. Thread = 2 adjacent time
// samples (one float4 load), lanes along time (coalesced); blockIdx.y = channel chunk.
// zap (optional): rows flagged by sk_decide_kernel are zeroed here (K15) instead of being added.
// Rows that are not 16-byte aligned (odd time_count, or an 8-byte aligned spectrum) take two float2 loads.
__global__ void __launch_bounds__(256) colsum_partial_kernel(float2* __restrict__ x,
                                                             size_t time_count, size_t chan_count,
                                                             size_t ts_count, size_t rows_per_chunk,
                                                             float* __restrict__ partial,
                                                             const unsigned char* __restrict__ zap) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t j2 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 2;
  if (j2 >= time_count) return;
  const size_t c0 = (size_t)blockIdx.y * rows_per_chunk;
  const size_t c1 = min(c0 + rows_per_chunk, chan_count);
  float a0 = 0.f, a1 = 0.f;
  const bool two = (j2 + 1 < time_count);
  const bool vec = ((time_count & 1) == 0) && aligned16(x);  // then every row, and j2, is 16-byte aligned
  if (vec && two) {
#pragma unroll 8
    for (size_t c = c0; c < c1; c++) {
      float4* p = reinterpret_cast<float4*>(x + c * time_count + j2);
      if (zap && zap[c]) {
        *p = make_float4(0.f, 0.f, 0.f, 0.f);
        continue;
      }
      const float4 v = *p;
      a0 += v.x * v.x + v.y * v.y;
      a1 += v.z * v.z + v.w * v.w;
    }
  } else {
    for (size_t c = c0; c < c1; c++) {
      if (zap && zap[c]) {
        x[c * time_count + j2] = make_float2(0.f, 0.f);
        if (two) x[c * time_count + j2 + 1] = make_float2(0.f, 0.f);
        continue;
      }
      const float2 v = x[c * time_count + j2];
      a0 += v.x * v.x + v.y * v.y;
      if (two) {
        const float2 w = x[c * time_count + j2 + 1];
        a1 += w.x * w.x + w.y * w.y;
      }
    }
  }
  if (j2 < ts_count) {
    float* p = partial + (size_t)blockIdx.y * ts_count + j2;
    p[0] = a0;
    if (j2 + 1 < ts_count) p[1] = a1;
  }
}

// K17 stage 2 + K16 + K18 + K20 in one launch: ts[j] = sum over chunks (fixed order) and zero_count by every CTA
// (CTA = 32 columns x 32 chunk groups: coalesced along time, fixed-order tree over the groups); the LAST CTA to
// finish (ticket) then removes the mean, forms the inclusive scan (fp64 carries) and fills the result header —
// what used to be a separate single-CTA kernel between two launches.
__global__ void __launch_bounds__(1024) colsum_final_scan_kernel(const float* __restrict__ partial,
                                                                 size_t ts_count, size_t chunks,
                                                                 float* __restrict__ ts, float* __restrict__ acc,
                                                                 const float2* __restrict__ x,
                                                                 size_t time_count, size_t chan_count,
                                                                 float chan_thr, size_t max_boxcar,
                                                                 unsigned* __restrict__ ticket,
                                                                 detect_dev_result* __restrict__ res,
                                                                 size_t ts_trial_stride, size_t acc_trial_stride,
                                                                 float* __restrict__ raw) {
  __shared__ float sm[32][33];
  __shared__ double smd[32];
  __shared__ double warp_tot[32];
  __shared__ float s_mean;
  __shared__ bool s_last;
  pdl_launch_dependents();
  pdl_wait();
  const int tid = threadIdx.x, lx = tid & 31, ly = tid >> 5;
  // batched over trials (incoherent DM search): blockIdx.y selects the trial's series, scan, ticket and header; the
  // block path launches one row of CTAs, so y = 0
  {
    const size_t y = blockIdx.y;
    if (partial) partial += y * chunks * ts_count;
    ts += y * ts_trial_stride;
    acc += y * acc_trial_stride;
    ticket += y;
    res += y;
  }
  // one wave of CTAs, each walking its share of the 32-column groups: the grid-wide fence + ticket at the end then
  // costs one round of latency instead of one per wave. The partial rows of a group are loaded eight at a time
  // (independent loads in flight) and added in index order. partial == nullptr: ts already holds the series
  // (the incoherent search writes it there), only the zero count, mean removal and scan run. raw (optional, y = 0
// only): also receives the un-centred column sums (the total-intensity sum of stream_sum.cuh adds them).
  const size_t per = (chunks + 31) / 32;
  const size_t c0 = (size_t)ly * per, c1 = min(c0 + per, chunks);
  for (size_t grp = blockIdx.x; partial && grp * 32 < ts_count; grp += gridDim.x) {
    const size_t j = grp * 32 + lx;
    float a = 0.f;
    if (j < ts_count) {
      for (size_t c = c0; c < c1; c += 8) {
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; u++) v[u] = (c + u < c1) ? partial[(c + u) * ts_count + j] : 0.f;
#pragma unroll
        for (int u = 0; u < 8; u++) a += v[u];
      }
    }
    __syncthreads();  // sm[][] of the previous group has been consumed
    sm[ly][lx] = a;
    __syncthreads();
    if (ly == 0 && j < ts_count) {
      float t = sm[0][lx];
#pragma unroll
      for (int g = 1; g < 32; g++) t += sm[g][lx];
      ts[j] = t;
      if (raw) raw[j] = t;
    }
  }
  // K16: channels whose first sample is zero; every CTA takes a slice, integer atomics (exact)
  {
    const size_t c = (size_t)blockIdx.x * blockDim.x + tid;
    int z = 0;
    if (c < chan_count) {
      const float2 v = x[c * time_count];
      z = (v.x * v.x + v.y * v.y == 0.f) ? 1 : 0;
    }
    const unsigned m = __ballot_sync(0xffffffffu, z);
    if (lx == 0 && m) atomicAdd(&res->zero_count, (unsigned long long)__popc(m));
    for (size_t cc = c + (size_t)gridDim.x * blockDim.x; cc < chan_count; cc += (size_t)gridDim.x * blockDim.x) {
      const float2 v = x[cc * time_count];
      if (v.x * v.x + v.y * v.y == 0.f) atomicAdd(&res->zero_count, 1ull);
    }
  }
  // ---- last CTA: mean removal, inclusive scan, header. One fence per CTA: the barrier orders every thread's stores
  // before thread 0's fence, which is cumulative (PTX memory model), so they are visible to whoever sees the ticket
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
    if (s_last) __threadfence();  // acquiring side, once: 32 warps fencing one after the other cost ~30 us here
  }
  __syncthreads();
  if (!s_last) return;
  const int nt = blockDim.x;
  // every access below is a 16-byte vector per thread (a warp touches 512 contiguous bytes): a single CTA that
  // scatters 4-byte accesses over 32 sectors per instruction spends a microsecond per thousand of them
  const bool vec = ((reinterpret_cast<uintptr_t>(ts) | reinterpret_cast<uintptr_t>(acc)) & 15u) == 0;
  auto load4 = [&](size_t i0, float (&v)[4]) {
    if (vec && i0 + 3 < ts_count) {
      const float4 q = __ldcg(reinterpret_cast<const float4*>(ts + i0));
      v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    } else {
#pragma unroll
      for (int e = 0; e < 4; e++) v[e] = (i0 + e < ts_count) ? __ldcg(&ts[i0 + e]) : 0.f;
    }
  };
  double local = 0.0;
  for (size_t i0 = (size_t)4 * tid; i0 < ts_count; i0 += (size_t)4 * nt) {
    float v[4];
    load4(i0, v);
    local += ((double)v[0] + (double)v[1]) + ((double)v[2] + (double)v[3]);
  }
  const double total = block_sum<double>(local, smd);
  if (tid == 0) s_mean = (float)total / (float)ts_count;   // map_average: sum / float(count)
  __syncthreads();
  const float mean = s_mean;
  // inclusive scan in tiles of 4 * blockDim.x elements: a thread scans its four in fp64, one block-wide exclusive
  // scan of the thread totals (warp shuffles, then the 32 warp totals) supplies the offsets, `carry` links the tiles
  double carry = 0.0;
  const size_t tile = (size_t)4 * nt;
  for (size_t base = 0; base < ts_count; base += tile) {
    const size_t i0 = base + (size_t)4 * tid;
    float v[4];
    load4(i0, v);
#pragma unroll
    for (int e = 0; e < 4; e++) v[e] = (i0 + e < ts_count) ? v[e] - mean : 0.f;
    const double t = ((double)v[0] + (double)v[1]) + ((double)v[2] + (double)v[3]);
    double incl = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lx >= o) incl += u;
    }
    if (lx == 31) warp_tot[ly] = incl;
    __syncthreads();
    if (ly == 0) {
      const double w = warp_tot[lx];
      double wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const double u = __shfl_up_sync(0xffffffffu, wi, o);
        if (lx >= o) wi += u;
      }
      warp_tot[lx] = wi - w;                 // exclusive offset of warp lx
      if (lx == 31) smd[0] = wi;             // tile total
    }
    __syncthreads();
    double run = carry + warp_tot[ly] + (incl - t);
    float a4[4];
#pragma unroll
    for (int e = 0; e < 4; e++) {
      run += (double)v[e];
      a4[e] = (float)run;
    }
    if (vec && i0 + 3 < ts_count) {
      *reinterpret_cast<float4*>(ts + i0) = make_float4(v[0], v[1], v[2], v[3]);
      *reinterpret_cast<float4*>(acc + i0) = make_float4(a4[0], a4[1], a4[2], a4[3]);
    } else {
#pragma unroll
      for (int e = 0; e < 4; e++)
        if (i0 + e < ts_count) {
          ts[i0 + e] = v[e];
          acc[i0 + e] = a4[e];
        }
    }
    carry += smd[0];
    __syncthreads();
  }
  if (tid == 0) {
    res->time_series_count = ts_count;
    const unsigned long long zc = *reinterpret_cast<volatile unsigned long long*>(&res->zero_count);  // all CTAs' atomics
    const int enabled = ((float)zc < chan_thr * (float)chan_count) ? 1 : 0;
    res->detect_enabled = enabled;
    int nb = 0;
    if (enabled) {
      nb = 1;
      for (size_t b = 2; b <= max_boxcar && b < ts_count && nb < 32; b *= 2) nb++;
    }
    res->n_boxcars = nb;
    *ticket = 0;
  }
}

// K19 + K21: one CTA per boxcar length 2^blockIdx.x: series, variance, threshold, count.
// host_out (optional): pinned host memory [MAX_BOXCARS][row_stride] that receives, straight from this kernel, the
// series of every boxcar with a positive count — the reference attaches the host copy of a series to the work only
// when count_signal is positive (signal_detect_pipe.hpp:347-366,405-423); negative blocks cost no PCIe traffic.
// gridDim.y > 1 runs one trial per y (series, acc, res and peak advanced by the given strides and one record).
// PEAK (DM sweep): the counting pass also reduces (max v[j], smallest j reaching it) and writes peak->snr[nb] =
// max / sqrt(variance) (0 when the variance is 0) and peak->peak_index[nb]; the block path launches PEAK = false.
template <bool PEAK = false>
__global__ void __launch_bounds__(1024) detect_boxcar_kernel(float* __restrict__ series, size_t row_stride,
                                                             const float* __restrict__ acc,
                                                             size_t ts_count, float snr,
                                                             detect_dev_result* __restrict__ res,
                                                             float* __restrict__ host_out,
                                                             detect_dev_peak* __restrict__ peak,
                                                             size_t series_trial_stride, size_t acc_trial_stride) {
  __shared__ double smd[32];
  __shared__ float s_thr;
  pdl_launch_dependents();
  pdl_wait();
  {  // batched over trials (incoherent DM search, host_out == nullptr there): blockIdx.y = trial; else y = 0
    const size_t y = blockIdx.y;
    series += y * series_trial_stride;
    acc += y * acc_trial_stride;
    res += y;
    if (PEAK) peak += y;
  }
  const int nb = blockIdx.x;
  if (nb >= res->n_boxcars) return;
  const int tid = threadIdx.x, nt = blockDim.x;
  const size_t b = (size_t)1 << nb;
  float* v = series + (size_t)nb * row_stride;
  const size_t n = (nb == 0) ? ts_count : ts_count - b;
  // eight independent loads in flight per thread and pass (a single CTA per boxcar is latency bound otherwise)
  double sq = 0.0;
  for (size_t i = tid; i < n; i += (size_t)8 * nt) {
    float d[8];
#pragma unroll
    for (int e = 0; e < 8; e++) {
      const size_t j = i + (size_t)e * nt;
      d[e] = (j < n) ? ((nb == 0) ? v[j] : acc[j + b] - acc[j]) : 0.f;
    }
#pragma unroll
    for (int e = 0; e < 8; e++) {
      const size_t j = i + (size_t)e * nt;
      if (nb != 0 && j < n) v[j] = d[e];
      sq += (double)d[e] * (double)d[e];
    }
  }
  sq = block_sum<double>(sq, smd);
  if (tid == 0) {
    const float var = (float)sq / (float)n;
    s_thr = snr * sqrtf(var);
    res->variance[nb] = var;
    res->threshold[nb] = s_thr;
    res->boxcar_length[nb] = b;
    res->series_length[nb] = n;
  }
  __syncthreads();
  const float thr = s_thr;
  double cnt = 0.0;
  float pv = -INFINITY;      // PEAK: this thread's largest value and the smallest index holding it
  unsigned long long pi = ~0ull;
  for (size_t i = tid; i < n; i += (size_t)8 * nt) {
    float d[8];
#pragma unroll
    for (int e = 0; e < 8; e++) {
      const size_t j = i + (size_t)e * nt;
      d[e] = (j < n) ? v[j] : -INFINITY;
    }
#pragma unroll
    for (int e = 0; e < 8; e++) {
      if (d[e] > thr) cnt += 1.0;
      if constexpr (PEAK) {
        // a thread visits its indices in increasing order, so a strict > keeps the first one of a tie
        const size_t j = i + (size_t)e * nt;
        if (j < n && (d[e] > pv || pi == ~0ull)) {
          pv = d[e];
          pi = j;
        }
      }
    }
  }
  cnt = block_sum<double>(cnt, smd);
  if (tid == 0) res->signal_count[nb] = (unsigned long long)cnt;
  if constexpr (PEAK) {
    // (value, index) reduction: larger value wins, equal values take the smaller index; any order gives one answer
    auto better = [](float av, unsigned long long ai, float bv, unsigned long long bi) {
      if (bi == ~0ull) return false;
      if (ai == ~0ull) return true;
      return bv > av || (bv == av && bi < ai);
    };
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_down_sync(0xffffffffu, pv, o);
      const unsigned long long oi = __shfl_down_sync(0xffffffffu, pi, o);
      if (better(pv, pi, ov, oi)) {
        pv = ov;
        pi = oi;
      }
    }
    __shared__ float s_pv[32];
    __shared__ unsigned long long s_pi[32];
    const int lane = tid & 31, wid = tid >> 5;
    if (lane == 0) {
      s_pv[wid] = pv;
      s_pi[wid] = pi;
    }
    __syncthreads();
    if (wid == 0) {
      pv = (lane < (nt + 31) / 32) ? s_pv[lane] : -INFINITY;
      pi = (lane < (nt + 31) / 32) ? s_pi[lane] : ~0ull;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_down_sync(0xffffffffu, pv, o);
        const unsigned long long oi = __shfl_down_sync(0xffffffffu, pi, o);
        if (better(pv, pi, ov, oi)) {
          pv = ov;
          pi = oi;
        }
      }
      if (lane == 0) {
        const float var = res->variance[nb];
        peak->snr[nb] = (var > 0.f && pi != ~0ull) ? pv / sqrtf(var) : 0.f;
        peak->peak_index[nb] = (pi != ~0ull) ? pi : 0ull;
      }
    }
  }
  if (host_out) {
    __shared__ int s_hit;
    if (tid == 0) s_hit = cnt > 0.0 ? 1 : 0;
    __syncthreads();
    if (s_hit) {
      float* h = host_out + (size_t)nb * row_stride;
      for (size_t i = tid; i < n; i += nt) h[i] = v[i];
      __syncthreads();
      if (tid == 0) __threadfence_system();
    }
  }
}

// ---- alternates of the refft path (spectra laid out [time][frequency]; SURVEY 8 f-4) ----------------------------
// spectral kurtosis v1 (spectrum/rfi_mitigation.hpp:181-275, normalization = false): per FREQUENCY column j over the
// time_counts spectra, s2 = sum |x|^2, s4 = sum |x|^4, sk = M s4 / s2^2; columns outside the thresholds are zeroed.
// Block (32, 8): lanes along frequency (coalesced), eight time phases per column folded in a fixed order.
__global__ void __launch_bounds__(256) sk_v1_stats_kernel(const float2* __restrict__ x, size_t fft_bins, size_t time_counts,
                                                          float thr_lo, float thr_hi, unsigned char* __restrict__ zap,
                                                          float* __restrict__ sk_out) {
  __shared__ float p2[8][33], p4[8][33];
  const int cx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const size_t j = (size_t)blockIdx.x * 32 + cx;
  float s2 = 0.f, s4 = 0.f;
  if (j < fft_bins) {
    for (size_t i = ty; i < time_counts; i += 8) {
      const float2 v = x[i * fft_bins + j];
      const float x2 = v.x * v.x + v.y * v.y;
      s2 += x2;
      s4 += x2 * x2;
    }
  }
  p2[ty][cx] = s2;
  p4[ty][cx] = s4;
  __syncthreads();
  if (ty == 0 && j < fft_bins) {
    float a = p2[0][cx], b = p4[0][cx];
#pragma unroll
    for (int g = 1; g < 8; g++) {
      a += p2[g][cx];
      b += p4[g][cx];
    }
    const float sk = (float)time_counts * (b / (a * a));
    zap[j] = (sk > thr_hi || sk < thr_lo) ? 1 : 0;  // NaN (an all-zero column): untouched
    if (sk_out) sk_out[j] = sk;
  }
}

__global__ void __launch_bounds__(256) sk_v1_zero_kernel(float2* __restrict__ x, size_t fft_bins, size_t time_counts,
                                                         const unsigned char* __restrict__ zap) {
  const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= fft_bins || !zap[j]) return;
  for (size_t i = blockIdx.y; i < time_counts; i += gridDim.y) x[i * fft_bins + j] = make_float2(0.f, 0.f);
}

// signal_detect_pipe v1 (pipeline/signal_detect_pipe.hpp:101-117): one value per spectrum = sum over its frequency bins
// of |x|^2 (multi_mapreduce with one work group per spectrum). One warp per spectrum, fixed shuffle tree.
__global__ void __launch_bounds__(256) rowsum_norm_kernel(const float2* __restrict__ x, size_t count_per_batch,
                                                          size_t batch_size, float* __restrict__ out) {
  const size_t row = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= batch_size) return;
  const int lane = threadIdx.x & 31;
  const float2* const p = x + row * count_per_batch;
  float a = 0.f;
  for (size_t j = lane; j < count_per_batch; j += 32) {
    const float2 v = p[j];
    a += v.x * v.x + v.y * v.y;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if (lane == 0) out[row] = a;
}

}  // namespace srtb_b200
