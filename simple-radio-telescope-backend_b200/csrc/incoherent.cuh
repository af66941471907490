// incoherent.cuh — semi-coherent DM search on one stream's dynamic spectrum (srtb_b200_incoherent_dm_search).
//
// The block path leaves x[C][L], coherently dedispersed at `dm`. For a trial DM_d near dm, the residual dispersion
// between channels is a whole-sample delay s[d][c] of the dynamic spectrum; the trial's series is
//
//   v_d[j] = sum_c |x[c][j + S- + s[d][c]]|^2,   j < T = ts - S+ - S-,
//
// in fp32, the channels added in index order (deterministic). One kernel forms every trial's series:
//
//   incoherent_dedisperse_kernel  a CTA owns a time tile of INC_TILE outputs and a group of up to INC_GROUP trials.
//                                 For each channel it stages the power of the span the group's shifts reach,
//                                 tile + max s - min s over the group, in shared memory: raw float2 through cp.async
//                                 (three buffers: the next two channels' copies run under this channel's adds), then
//                                 |x|^2 once per staged sample. Each thread keeps 4 trials x 8 times in registers.
//
// The host sorts the trials by DM and cuts the sorted list into groups whose shift spread fits the staging buffer, so
// neighbouring trials (small spread) share a group and trials need not be given in order. The detector's tail then
// runs batched over the trials (colsum_final_scan_kernel and detect_boxcar_kernel with blockIdx.y = trial).
#pragma once
#include <cuda_runtime.h>

#include "ops_kernels.cuh"

namespace srtb_b200 {

constexpr int INC_TILE = 256;    // time outputs per CTA
constexpr int INC_GROUP = 64;    // trials per CTA, at most
constexpr int INC_THREADS = 512; // 16 warps: warp w adds trials w, w + 16, w + 32, w + 48
constexpr int INC_SPREAD_MAX = 1792;  // largest shift spread of a group: staging buffer of INC_TILE + 1792 samples
constexpr int INC_STAGES = 3;         // channels in flight: this one and the next two

// dynamic shared memory of a launch whose groups spread at most `spread` samples
__host__ __device__ constexpr size_t incoherent_smem_bytes(unsigned spread) {
  return (size_t)(INC_TILE + spread) * (INC_STAGES * sizeof(float2) + sizeof(float)) +
         INC_STAGES * INC_GROUP * sizeof(int);
}

__device__ __forceinline__ void cp_async8(void* smem_dst, const void* gmem_src, bool valid) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  const int n = valid ? 8 : 0;  // 0: zero-fill, nothing is read
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(d), "l"(gmem_src), "r"(n) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gmem_src) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait2() { asm volatile("cp.async.wait_group 2;\n" ::: "memory"); }

// x: [C][L] complex64, 8-byte aligned. off: [C][n_dm] absolute offsets s + S- (>= 0) of each trial, the trials in
// sorted order; gspan: [groups][C] (min, max) of off over the group's trials; groups: [groups] (first sorted slot,
// trial count); order: [n_dm] trial index of each sorted slot. span_max = INC_TILE + the largest spread.
// out: trial d's series [T] at out + d * out_stride. Grid: (groups, min(tiles, 65535)) with tiles = ceil(T / INC_TILE);
// CTA y forms tiles y, y + gridDim.y, ... in turn, so T may exceed 65535 tiles (gridDim.y's limit, T just above 2^24).
__global__ void __launch_bounds__(INC_THREADS) incoherent_dedisperse_kernel(
    const float2* __restrict__ x, size_t L, size_t C, size_t T, size_t n_dm, const int* __restrict__ off,
    const int2* __restrict__ gspan, const int2* __restrict__ groups, const int* __restrict__ order, unsigned span_max,
    float* __restrict__ out, size_t out_stride) {
  extern __shared__ __align__(16) unsigned char inc_smem[];
  float2* raw = reinterpret_cast<float2*>(inc_smem);                          // [INC_STAGES][span_max]
  float* pw = reinterpret_cast<float*>(raw + INC_STAGES * (size_t)span_max);  // [span_max]
  int* s_off = reinterpret_cast<int*>(pw + span_max);                        // [INC_STAGES][INC_GROUP]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const size_t g = blockIdx.x;
  const int2 gi = groups[g];
  const int cnt = gi.y;
  const int* goff = off + gi.x;
  const int2* gsp = gspan + g * C;
  const size_t tiles = (T + INC_TILE - 1) / INC_TILE;

  for (size_t tile = blockIdx.y; tile < tiles; tile += gridDim.y) {  // CTA-uniform
    const size_t t0 = tile * INC_TILE;

    // channel c's span -> raw[c % 3], its slot offsets -> s_off[c % 3]; one commit group per channel. The previous
    // tile read raw and s_off only before its last channel's second barrier, so restaging them here is safe
    auto stage = [&](size_t c) {
      const int2 mm = gsp[c];
      const size_t span = INC_TILE + (size_t)(mm.y - mm.x);
      const float2* row = x + c * L;
      const size_t src0 = t0 + (size_t)mm.x;
      float2* dst = raw + (c % INC_STAGES) * (size_t)span_max;
      for (size_t e = tid; e < span; e += INC_THREADS) {
        const bool valid = src0 + e < L;
        cp_async8(dst + e, valid ? row + src0 + e : row, valid);
      }
      if (tid < cnt) cp_async4(s_off + (c % INC_STAGES) * INC_GROUP + tid, goff + c * n_dm + tid);
      cp_async_commit();
    };

    float acc[4][8];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
      for (int r = 0; r < 8; r++) acc[i][r] = 0.f;

    stage(0);
    if (C > 1) stage(1);
    else cp_async_commit();
    for (size_t c = 0; c < C; c++) {
      if (c + 2 < C) stage(c + 2);
      else cp_async_commit();  // empty groups keep wait_group 2 meaning "channel c has landed"
      cp_async_wait2();
      __syncthreads();  // channel c visible to all; every warp is done with the previous channel's (or tile's) pw
      const int2 mm = gsp[c];
      const size_t span = INC_TILE + (size_t)(mm.y - mm.x);
      const float2* src = raw + (c % INC_STAGES) * (size_t)span_max;
      for (size_t e = tid; e < span; e += INC_THREADS) {
        const float2 v = src[e];
        pw[e] = __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y));
      }
      // this channel's offsets are read before the barrier: the next iteration's stage() overwrites s_off[c % 3]
      int rel[4];
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int k = warp + 16 * i;
        rel[i] = (k < cnt) ? s_off[(c % INC_STAGES) * INC_GROUP + k] - mm.x : 0;
      }
      __syncthreads();
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int k = warp + 16 * i;
        if (k < cnt) {  // warp-uniform
          const float* p = pw + rel[i] + lane;
#pragma unroll
          for (int r = 0; r < 8; r++) acc[i][r] += p[32 * r];
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int k = warp + 16 * i;
      if (k >= cnt) continue;
      float* o = out + (size_t)order[gi.x + k] * out_stride;
#pragma unroll
      for (int r = 0; r < 8; r++) {
        const size_t j = t0 + lane + 32 * r;
        if (j < T) o[j] = acc[i][r];
      }
    }
  }
}

}  // namespace srtb_b200
