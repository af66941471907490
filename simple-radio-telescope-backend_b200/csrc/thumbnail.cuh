// thumbnail.cuh — the waterfall thumbnail of simplify_spectrum_pipe_2 (S/pipeline/spectrum_pipe.hpp:82-143):
// resample_spectrum_3 with norm() (S/spectrum/simplify_spectrum.hpp:423-620), then
// simplify_spectrum_normalize_with_average_value (:627-644) and generate_pixmap (:700-731), as three kernels:
//
//   thumb_row_kernel   reads the [C][L] complex64 spectrum once (coalesced 16-byte loads into shared memory) and
//                      writes R[C][W], every input row resampled along time, kept in L2 (evict-last);
//   thumb_col_kernel   out[y2][x2] = sum_y w_y R[y][x2] (coalesced along x2), plus one partial sum per CTA;
//   thumb_norm_kernel  folds the partials in a fixed order into the average (on the device, no host round trip),
//                      scales the intensities by 1 / (2 avg) when avg > FLT_EPSILON and writes the ARGB pixmap.
//
// Pixel edges, ceil/floor and the edge weights are the reference's fp32 expressions, evaluated with explicit
// round-to-nearest intrinsics (no contraction), so the integer ranges and weights are bit-identical to it. The sums
// are taken in another order than the reference's work-item split; no atomics, so every call gives the same bits.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace srtb_b200 {

// one output pixel's extent along one axis: cells [lo, hi) with weight 1, cell lo - 1 with weight wl (when wl > 0),
// cell hi with weight wh (when wh > 0). When the pixel lies inside one input cell, lo - 1 == hi and both edge terms
// apply to that cell, as in the reference (quirk q12: weight r - l + 1 instead of r - l).
struct thumb_extent {
  long long lo, hi;
  float wl, wh;
};

__device__ __forceinline__ thumb_extent thumb_edges(size_t i, float out_f, float in_f) {
  const float a = __fmul_rn(__fdiv_rn(__ull2float_rn(i), out_f), in_f);      // left_accurate
  const float b = __fmul_rn(__fdiv_rn(__ull2float_rn(i + 1), out_f), in_f);  // right_accurate
  const float lr = ceilf(a), hr = floorf(b);
  thumb_extent e;
  e.lo = (long long)lr;
  e.hi = (long long)hr;
  e.wl = lr > a ? __fsub_rn(lr, a) : 0.f;
  e.wh = b > hr ? __fsub_rn(b, hr) : 0.f;
  return e;
}
__device__ __forceinline__ long long thumb_first(const thumb_extent& e) { return e.wl > 0.f ? e.lo - 1 : e.lo; }
__device__ __forceinline__ long long thumb_end(const thumb_extent& e) { return e.wh > 0.f ? e.hi + 1 : e.hi; }

// |x|^2 as the reference's srtb::norm writes it (S/math.hpp:59-66), without contraction
__device__ __forceinline__ float thumb_norm(float re, float im) { return __fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im)); }

// this cell's contribution to the pixel of extent e, in the reference's term order (left edge, body, right edge)
__device__ __forceinline__ float thumb_add(float acc, long long c, const thumb_extent& e, float v) {
  if (e.wl > 0.f && c == e.lo - 1) acc = __fadd_rn(acc, __fmul_rn(e.wl, v));
  if (c >= e.lo && c < e.hi) acc = __fadd_rn(acc, v);
  if (e.wh > 0.f && c == e.hi) acc = __fadd_rn(acc, __fmul_rn(e.wh, v));
  return acc;
}

constexpr int THUMB_THREADS = 256;
constexpr int THUMB_CHUNK = 2048;  // input cells staged in shared memory at a time

__device__ __forceinline__ uint64_t thumb_evict_last_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}

// Row stage. Block (row y = blockIdx.x, pixel tile blockIdx.y): G consecutive threads share one output pixel x2
// (lane j adds the cells first + j, first + j + G, ...), so a CTA covers 256 / G pixels, whose input cells are one
// contiguous span of the row; the span is staged through shared memory in chunks. VEC: 16-byte loads (L even and the
// spectrum 16-byte aligned), else 8-byte loads; both are coalesced.
template <bool VEC>
__global__ void __launch_bounds__(THUMB_THREADS) thumb_row_kernel(const float2* __restrict__ spec, size_t L, size_t W,
                                                                  int G, float* __restrict__ rows) {
  __shared__ float cell[THUMB_CHUNK];
  const float in_f = __ull2float_rn(L), out_f = __ull2float_rn(W);
  const size_t y = blockIdx.x;
  const int per_cta = THUMB_THREADS / G;
  const size_t px0 = (size_t)blockIdx.y * per_cta;
  const size_t px1 = min(px0 + per_cta, W);
  const size_t x2 = px0 + threadIdx.x / G;
  const int lane = threadIdx.x % G;
  const bool live = x2 < px1;
  const thumb_extent e = thumb_edges(live ? x2 : px1 - 1, out_f, in_f);
  const long long span0 = max(thumb_first(thumb_edges(px0, out_f, in_f)), 0ll);
  const long long span1 = min(thumb_end(thumb_edges(px1 - 1, out_f, in_f)), (long long)L);
  const long long my0 = thumb_first(e) + lane;
  const long long my1 = thumb_end(e);
  const size_t base = y * L;
  float acc = 0.f;
  for (long long k0 = span0; k0 < span1; k0 += THUMB_CHUNK) {
    const long long k1 = min(k0 + THUMB_CHUNK, span1);
    if constexpr (VEC) {
      const float4* s4 = reinterpret_cast<const float4*>(spec);
      const size_t q0 = (base + (size_t)k0) >> 1, q1 = (base + (size_t)k1 + 1) >> 1;
      for (size_t q = q0 + threadIdx.x; q < q1; q += THUMB_THREADS) {
        const float4 v = __ldcs(s4 + q);
        const long long c = (long long)(2 * q - base);
        if (c >= k0) cell[c - k0] = thumb_norm(v.x, v.y);
        if (c + 1 < k1) cell[c + 1 - k0] = thumb_norm(v.z, v.w);
      }
    } else {
      for (long long c = k0 + threadIdx.x; c < k1; c += THUMB_THREADS) {
        const float2 v = __ldcs(spec + base + c);
        cell[c - k0] = thumb_norm(v.x, v.y);
      }
    }
    __syncthreads();
    if (live) {
      // the first of this lane's cells at or after k0
      long long c = my0 >= k0 ? my0 : my0 + ((k0 - my0 + G - 1) / G) * G;
      for (const long long end = min(my1, k1); c < end; c += G) acc = thumb_add(acc, c, e, cell[c - k0]);
    }
    __syncthreads();
  }
  // fixed-order reduction over the G lanes of the pixel (G is a power of two, the group lies inside one warp)
  for (int off = G >> 1; off > 0; off >>= 1) acc = __fadd_rn(acc, __shfl_down_sync(0xffffffffu, acc, off, G));
  if (live && lane == 0) {
    float* dst = rows + y * W + x2;
    asm volatile("st.global.L2::cache_hint.f32 [%0], %1, %2;" ::"l"(dst), "f"(acc), "l"(thumb_evict_last_policy())
                 : "memory");
  }
}

// fixed-order sum over the CTA (warp shuffles, then warp 0 over the warp sums); the result is valid in thread 0
__device__ __forceinline__ float thumb_block_sum(float v, float* red) {
  for (int off = 16; off > 0; off >>= 1) v = __fadd_rn(v, __shfl_down_sync(0xffffffffu, v, off));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    v = threadIdx.x < THUMB_THREADS / 32 ? red[threadIdx.x] : 0.f;
    for (int off = 16; off > 0; off >>= 1) v = __fadd_rn(v, __shfl_down_sync(0xffffffffu, v, off));
  }
  return v;
}

// Column stage: pixel i = y2 * W + x2 is taken by thread i of a grid-stride loop (coalesced along x2); the y terms
// are summed in the reference's order (top edge, body, bottom edge). partial[blockIdx.x] = this CTA's sum of out.
__global__ void __launch_bounds__(THUMB_THREADS) thumb_col_kernel(const float* __restrict__ rows, size_t C, size_t W,
                                                                  size_t H, float* __restrict__ out,
                                                                  float* __restrict__ partial) {
  __shared__ float red[THUMB_THREADS / 32];
  const float in_f = __ull2float_rn(C), out_f = __ull2float_rn(H);
  const size_t n = W * H;
  float local = 0.f;
  for (size_t i = (size_t)blockIdx.x * THUMB_THREADS + threadIdx.x; i < n; i += (size_t)gridDim.x * THUMB_THREADS) {
    const size_t y2 = i / W, x2 = i - y2 * W;
    const thumb_extent e = thumb_edges(y2, out_f, in_f);
    float v = 0.f;
    if (e.wl > 0.f) v = __fadd_rn(v, __fmul_rn(e.wl, rows[(size_t)(e.lo - 1) * W + x2]));
    for (long long y = e.lo; y < e.hi; y++) v = __fadd_rn(v, rows[(size_t)y * W + x2]);
    if (e.wh > 0.f) v = __fadd_rn(v, __fmul_rn(e.wh, rows[(size_t)e.hi * W + x2]));
    out[i] = v;
    local = __fadd_rn(local, v);
  }
  const float s = thumb_block_sum(local, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

__device__ __forceinline__ unsigned thumb_channel(uint32_t c0, uint32_t c1, int shift, float v, float one_minus_v) {
  const float a = __uint2float_rn((c0 >> shift) & 0xffu), b = __uint2float_rn((c1 >> shift) & 0xffu);
  return (__float2uint_rz(__fadd_rn(__fmul_rn(one_minus_v, a), __fmul_rn(v, b))) & 0xffu) << shift;
}

// Normalise + pixmap: every CTA folds the n_partial column-stage partials in the same fixed order (so all agree on
// avg), then scales its pixels in place and writes their ARGB32 colour.
__global__ void __launch_bounds__(THUMB_THREADS) thumb_norm_kernel(float* __restrict__ inten, size_t n,
                                                                   const float* __restrict__ partial, int n_partial,
                                                                   uint32_t c0, uint32_t c1, uint32_t c_over,
                                                                   uint32_t* __restrict__ pixmap,
                                                                   float* __restrict__ d_average) {
  __shared__ float red[THUMB_THREADS / 32];
  __shared__ float s_avg;
  float v = 0.f;
  for (int j = threadIdx.x; j < n_partial; j += THUMB_THREADS) v = __fadd_rn(v, partial[j]);
  const float total = thumb_block_sum(v, red);
  if (threadIdx.x == 0) s_avg = __fdiv_rn(total, __ull2float_rn(n));  // map_average: sum / count
  __syncthreads();
  const float avg = s_avg;
  if (d_average && blockIdx.x == 0 && threadIdx.x == 0) *d_average = avg;
  const float coeff = __fdiv_rn(1.0f, __fmul_rn(avg, 2.0f));
  const bool scale = avg > 1.1920928955078125e-7f;  // FLT_EPSILON
  for (size_t i = (size_t)blockIdx.x * THUMB_THREADS + threadIdx.x; i < n; i += (size_t)gridDim.x * THUMB_THREADS) {
    float x = inten[i];
    if (scale) {
      x = __fmul_rn(x, coeff);
      inten[i] = x;
    }
    uint32_t argb = c_over;
    if (0.f <= x && x <= 1.f) {
      const float u = __fsub_rn(1.f, x);
      argb = thumb_channel(c0, c1, 24, x, u) | thumb_channel(c0, c1, 16, x, u) | thumb_channel(c0, c1, 8, x, u) |
             thumb_channel(c0, c1, 0, x, u);
    }
    pixmap[i] = argb;
  }
}

}  // namespace srtb_b200
