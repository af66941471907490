// correlator.cuh — the two element-wise stages of the reference's baseband correlator (U/src/correlator.cpp:109-140):
//
//   cross_spectrum_kernel  y[i] = (norm X1[i]) conj(X2[i]), i < M                          (its step (1))
//   magnitude_kernel       out[i] = |y[i]|, after the backward C2C of y                     (its step (3))
//
// The forward R2C of each input and the backward C2C between the two stages are the FFT engine's (fft_engine.cuh).
// Both kernels are grid-stride, with no atomics. The cross spectrum uses SyclCPLX's float arithmetic in its order
// (scalar times complex scales each part, then (ac - bd, ad + bc) with d = -Im X2) through round-to-nearest intrinsics,
// so no contraction changes a bit: on identical spectra it is bit-identical to the reference's expression.
#pragma once
#include <cuda_runtime.h>

namespace srtb_b200 {

__device__ __forceinline__ float2 cross_bin(float2 x1, float2 x2, float norm) {
  const float a = __fmul_rn(x1.x, norm), b = __fmul_rn(x1.y, norm);
  const float c = x2.x, d = -x2.y;
  return make_float2(__fsub_rn(__fmul_rn(a, c), __fmul_rn(b, d)), __fadd_rn(__fmul_rn(a, d), __fmul_rn(b, c)));
}

// out may be a or b (the reference writes over X1): each bin is read before its own store, and no other bin's.
// VEC: a, b and out 16-byte aligned, two bins per access, odd M finished by the first thread; else 8-byte accesses.
template <bool VEC>
__global__ void __launch_bounds__(256) cross_spectrum_kernel(const float2* a, const float2* b, size_t M, float norm,
                                                             float2* out) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if constexpr (VEC) {
    const float4* a4 = reinterpret_cast<const float4*>(a);
    const float4* b4 = reinterpret_cast<const float4*>(b);
    float4* o4 = reinterpret_cast<float4*>(out);
    for (size_t i = gid; i < M / 2; i += stride) {
      const float4 x = a4[i], y = b4[i];
      const float2 lo = cross_bin(make_float2(x.x, x.y), make_float2(y.x, y.y), norm);
      const float2 hi = cross_bin(make_float2(x.z, x.w), make_float2(y.z, y.w), norm);
      o4[i] = make_float4(lo.x, lo.y, hi.x, hi.y);
    }
    if ((M & 1) && gid == 0) out[M - 1] = cross_bin(a[M - 1], b[M - 1], norm);
  } else {
    for (size_t i = gid; i < M; i += stride) out[i] = cross_bin(a[i], b[i], norm);
  }
}

// out[i] = hypotf(Re y[i], Im y[i]) into M floats (out of place). VEC: y 16-byte and out 8-byte aligned, two bins per
// access, odd M finished by the first thread.
template <bool VEC>
__global__ void __launch_bounds__(256) magnitude_kernel(const float2* __restrict__ y, size_t M,
                                                        float* __restrict__ out) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if constexpr (VEC) {
    const float4* y4 = reinterpret_cast<const float4*>(y);
    float2* o2 = reinterpret_cast<float2*>(out);
    for (size_t i = gid; i < M / 2; i += stride) {
      const float4 v = y4[i];
      o2[i] = make_float2(hypotf(v.x, v.y), hypotf(v.z, v.w));
    }
    if ((M & 1) && gid == 0) out[M - 1] = hypotf(y[M - 1].x, y[M - 1].y);
  } else {
    for (size_t i = gid; i < M; i += stride) out[i] = hypotf(y[i].x, y[i].y);
  }
}

}  // namespace srtb_b200
