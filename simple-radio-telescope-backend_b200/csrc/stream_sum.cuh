// stream_sum.cuh — the single-pulse detector on the total intensity of a multi-stream block (block config field
// signal_detect_sum_streams).
//
// Each stream s of the block leaves its dynamic spectrum x_s[C][L] and, from its detector's column-sum kernel, the raw
// (un-centred) column sums R_s[j] = sum_c |x_s[c][j]|^2, j < L'. Channel c is dropped when |x_s[c][0]|^2 == 0 in any
// stream (the zero_count proxy: SK and the manual zap leave such rows zero); K is the set of kept channels, and
//
//   v[j] = sum_{c in K} sum_s |x_s[c][j]|^2 = sum_s R_s[j] - sum_{c mismatched} sum_{s keeping c} |x_s[c][j]|^2,
//
// where a mismatched channel is dropped in some streams and kept in others (its kept rows must not reach the sum).
// Two kernels, then the detector's own tail (colsum_final_scan_kernel with partial == nullptr, detect_boxcar_kernel):
//
//   stream_sum_mask_kernel  one CTA: reads the first sample of every channel of every stream, writes the mask
//                           (1, 0) / (0, 0) per channel (the tail counts its zeros: the union count C - |K|) and the
//                           mismatched channels in increasing order with the streams that keep them.
//   stream_sum_kernel       one thread per j: adds R_0[j] .. R_{S-1}[j] in stream order, then subtracts the kept rows
//                           of every mismatched channel in list order, streams in order. fp32, fixed order: the same
//                           bits on any schedule.
#pragma once
#include <cuda_runtime.h>

#include "ops_kernels.cuh"

namespace srtb_b200 {

constexpr int SUM_MAX_STREAMS = 4;

struct stream_sum_inputs {
  const float2* x[SUM_MAX_STREAMS];  // the streams' dynamic spectra [C][L]
  const float* raw[SUM_MAX_STREAMS]; // their raw column sums, L' each
};

// mis[k] = (channel, bit s set when stream s keeps it) for k < *n_mis
__global__ void __launch_bounds__(1024) stream_sum_mask_kernel(stream_sum_inputs in, int streams, size_t time_count,
                                                               size_t chan_count, float2* __restrict__ mask,
                                                               uint2* __restrict__ mis, unsigned* __restrict__ n_mis) {
  __shared__ unsigned warp_cnt[32];
  __shared__ unsigned s_base;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) s_base = 0;
  __syncthreads();
  for (size_t c0 = 0; c0 < chan_count; c0 += blockDim.x) {
    const size_t c = c0 + tid;
    unsigned keep = 0;
    bool mismatched = false;
    if (c < chan_count) {
      // constant trip counts keep the pointer arrays in the parameter bank (no local-memory copy)
#pragma unroll
      for (int s = 0; s < SUM_MAX_STREAMS; s++) {
        if (s >= streams) break;
        const float2 v = in.x[s][c * time_count];
        if (v.x * v.x + v.y * v.y != 0.f) keep |= 1u << s;
      }
      mismatched = keep != 0 && keep != (1u << streams) - 1;
      mask[c] = make_float2(keep == (1u << streams) - 1 ? 1.f : 0.f, 0.f);
    }
    // order-preserving compaction of the mismatched channels
    const unsigned ballot = __ballot_sync(0xffffffffu, mismatched);
    if (lane == 0) warp_cnt[wid] = __popc(ballot);
    __syncthreads();
    unsigned before = s_base;
    for (int w = 0; w < wid; w++) before += warp_cnt[w];
    if (mismatched) mis[before + __popc(ballot & ((1u << lane) - 1))] = make_uint2((unsigned)c, keep);
    __syncthreads();
    if (tid == 0) {
      unsigned t = 0;
      for (int w = 0; w < (int)(blockDim.x >> 5); w++) t += warp_cnt[w];
      s_base += t;
    }
    __syncthreads();
  }
  if (tid == 0) *n_mis = s_base;
}

__global__ void __launch_bounds__(256) stream_sum_kernel(stream_sum_inputs in, int streams, size_t time_count,
                                                         size_t ts_count, const uint2* __restrict__ mis,
                                                         const unsigned* __restrict__ n_mis, float* __restrict__ v) {
  pdl_launch_dependents();
  pdl_wait();
  const unsigned nm = *n_mis;
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < ts_count; j += (size_t)gridDim.x * blockDim.x) {
    float a = in.raw[0][j];
#pragma unroll
    for (int s = 1; s < SUM_MAX_STREAMS; s++)
      if (s < streams) a += in.raw[s][j];
    for (unsigned k = 0; k < nm; k++) {
      const uint2 m = mis[k];
#pragma unroll
      for (int s = 0; s < SUM_MAX_STREAMS; s++)
        if (m.y & (1u << s)) {
          const float2 y = in.x[s][(size_t)m.x * time_count + j];
          a -= y.x * y.x + y.y * y.y;
        }
    }
    v[j] = a;
  }
}

}  // namespace srtb_b200
