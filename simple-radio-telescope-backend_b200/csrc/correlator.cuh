// correlator.cuh — the two element-wise stages of the reference's baseband correlator (U/src/correlator.cpp:109-140):
//
//   cross_spectrum_kernel  y[i] = (norm X1[i]) conj(X2[i]), i < M                          (its step (1))
//   magnitude_kernel       out[i] = |y[i]|, after the backward C2C of y                     (its step (3))
//
// The forward R2C of each input and the backward C2C between the two stages are the FFT engine's (fft_engine.cuh).
// Both kernels are grid-stride, with no atomics. The cross spectrum uses SyclCPLX's float arithmetic in its order
// (scalar times complex scales each part, then (ac - bd, ad + bc) with d = -Im X2) through round-to-nearest intrinsics,
// so no contraction changes a bit: on identical spectra it is bit-identical to the reference's expression.
//
// The integrating, segment-averaged mode (srtb_b200_correlate_accumulate / _finish) adds three kernels:
//
//   corr_pack_kernel            two consecutive segments of one input -> one complex row x[2j] + i x[2j+1]
//   corr_split_accumulate_kernel  per bin k < Ms: split Z[k], conj Z[-k] into the two segments' bins, add
//                               X1_even conj(X2_even) + X1_odd conj(X2_odd) over the call's rows into a float64 sum
//   corr_scale_kernel           y[k] = complex64(acc[k] * norm / K), before the backward C2C and magnitude_kernel
//
// Between pack and split runs one batched forward C2C of length Ls over the rows of both inputs (fft_c2c_impl).
// Two segments of the same input share a row, not the two inputs: a stationary input's segments have similar levels,
// so the split's rounding error stays relative to each segment's own spectrum even when the inputs' levels differ.
#pragma once
#include <cuda_runtime.h>

#include "ops_kernels.cuh"

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

// ---- the integrating mode. Layout of the rows: out[s][j][t], s = input, j < rows = ceil(n_segments / 2), t < Ls =
// 2^log_ls; row j of input s holds x_s[2j Ls + t] + i x_s[(2j + 1) Ls + t], with a zero imaginary part when segment
// 2j + 1 does not exist (odd n_segments).
//
// VEC: each thread decodes 8 samples of the even and 8 of the odd segment with unpack_src<> (the inputs aligned to the
// 8-sample group, |BITS| bytes) and stores 4 float4. Else one sample pair per thread through unpack_one<>. Decoding is
// exact, so both routes give identical bits.
template <int BITS, bool VEC>
__global__ void __launch_bounds__(256) corr_pack_kernel(const void* __restrict__ in_1, const void* __restrict__ in_2,
                                                        int log_ls, size_t n_segments, size_t rows,
                                                        float2* __restrict__ out) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int log_item = VEC ? log_ls - 3 : log_ls;  // items per row: groups of 8 samples, or samples
  const size_t per_input = rows << log_item;
  for (size_t w = gid; w < 2 * per_input; w += stride) {
    const int s = w >= per_input;
    const size_t r = w - (s ? per_input : 0);
    const size_t j = r >> log_item, u = r & (((size_t)1 << log_item) - 1);
    const void* in = s ? in_2 : in_1;
    const bool odd = 2 * j + 1 < n_segments;
    float2* row = out + ((s ? rows : 0) + j) * ((size_t)1 << log_ls);
    if constexpr (VEC) {
      const size_t g = ((2 * j) << log_item) + u;  // first group of the even segment's 8 samples
      float e[8], o[8] = {};
      unpack_src<BITS>::get(in, g, e);
      if (odd) unpack_src<BITS>::get(in, g + ((size_t)1 << log_item), o);
      float4* dst = reinterpret_cast<float4*>(row + 8 * u);
#pragma unroll
      for (int q = 0; q < 4; q++) dst[q] = make_float4(e[2 * q], o[2 * q], e[2 * q + 1], o[2 * q + 1]);
    } else {
      const size_t i = ((2 * j) << log_ls) + u;
      row[u] = make_float2(unpack_one<BITS>(in, i), odd ? unpack_one<BITS>(in, i + ((size_t)1 << log_ls)) : 0.f);
    }
  }
}

__device__ __forceinline__ double2 mul_conj(double2 p, double2 q) {
  return make_double2(p.x * q.x + p.y * q.y, p.y * q.x - p.x * q.y);
}

// z: the forward-transformed rows of corr_pack_kernel. A CTA of 256 threads covers BT = 2^log_bt bins (BT = min(Ms,
// 256)) and 256 / BT row lanes; blockIdx.y is a group of rows_per_group rows. Each thread sums its rows in float64 in
// row order, the CTA adds its lanes in lane order, and so each (group, bin) sum is fixed by the shapes alone.
// One group (gridDim.y == 1): the CTA adds its sum into acc (or overwrites acc when reset). Several groups: each CTA
// stores its sum in partial[group][bin]; the last CTA of a bin tile to finish (per-tile ticket, reset by that CTA)
// adds the groups in group order into acc. The result is deterministic whatever order the CTAs run in.
__global__ void __launch_bounds__(256) corr_split_accumulate_kernel(const float2* __restrict__ z, int log_ls, int log_bt,
                                                                    size_t rows, size_t n_segments,
                                                                    size_t rows_per_group, double2* partial,
                                                                    unsigned* tickets, double2* acc, int reset) {
  __shared__ double2 red[256];
  __shared__ bool last;
  const size_t Ls = (size_t)1 << log_ls, Ms = Ls / 2, BT = (size_t)1 << log_bt;
  const unsigned lane = threadIdx.x >> log_bt, lanes = 256u >> log_bt;
  const size_t k = (size_t)blockIdx.x * BT + (threadIdx.x & (BT - 1));
  const size_t mk = (Ls - k) & (Ls - 1);  // the mirrored bin, -k mod Ls (k = 0 mirrors onto itself)
  const float2* z2 = z + rows * Ls;       // input 2's rows
  const size_t j_end = min(rows, ((size_t)blockIdx.y + 1) * rows_per_group);
  double2 sum = make_double2(0.0, 0.0);
  for (size_t j = (size_t)blockIdx.y * rows_per_group + lane; j < j_end; j += lanes) {
    const float2 a = z[j * Ls + k], b = z[j * Ls + mk], c = z2[j * Ls + k], d = z2[j * Ls + mk];
    // even segment: (Z[k] + conj Z[-k]) / 2; odd segment: (Z[k] - conj Z[-k]) / (2i)
    const double2 e1 = make_double2(0.5 * ((double)a.x + b.x), 0.5 * ((double)a.y - b.y));
    const double2 e2 = make_double2(0.5 * ((double)c.x + d.x), 0.5 * ((double)c.y - d.y));
    const double2 ee = mul_conj(e1, e2);
    sum.x += ee.x;
    sum.y += ee.y;
    if (2 * j + 1 < n_segments) {
      const double2 o1 = make_double2(0.5 * ((double)a.y + b.y), -0.5 * ((double)a.x - b.x));
      const double2 o2 = make_double2(0.5 * ((double)c.y + d.y), -0.5 * ((double)c.x - d.x));
      const double2 oo = mul_conj(o1, o2);
      sum.x += oo.x;
      sum.y += oo.y;
    }
  }
  red[threadIdx.x] = sum;
  __syncthreads();
  if (lane == 0) {
    for (unsigned l = 1; l < lanes; l++) {
      sum.x += red[l * BT + threadIdx.x].x;
      sum.y += red[l * BT + threadIdx.x].y;
    }
  }
  if (gridDim.y == 1) {
    if (lane == 0) acc[k] = reset ? sum : make_double2(acc[k].x + sum.x, acc[k].y + sum.y);
    return;
  }
  if (lane == 0) partial[(size_t)blockIdx.y * Ms + k] = sum;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(&tickets[blockIdx.x], 1u) == gridDim.y - 1;
  __syncthreads();
  if (!last) return;
  if (lane == 0) {
    double2 t = reset ? make_double2(0.0, 0.0) : acc[k];
    double2 g = make_double2(0.0, 0.0);
    for (unsigned y = 0; y < gridDim.y; y++) {
      const double2 p = __ldcg(&partial[(size_t)y * Ms + k]);
      g.x += p.x;
      g.y += p.y;
    }
    t.x += g.x;
    t.y += g.y;
    acc[k] = t;
  }
  if (threadIdx.x == 0) tickets[blockIdx.x] = 0;
}

// y[k] = complex64(acc[k] * scale), scale = norm / K in float64
__global__ void __launch_bounds__(256) corr_scale_kernel(const double2* __restrict__ acc, size_t Ms, double scale,
                                                         float2* __restrict__ y) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < Ms; k += stride)
    y[k] = make_float2((float)(acc[k].x * scale), (float)(acc[k].y * scale));
}

}  // namespace srtb_b200
