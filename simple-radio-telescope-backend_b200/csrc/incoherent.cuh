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
// The staging and accumulation of one tile (inc_tile) is a template over the rows it reads, so the candidate cut-outs'
// DM-time plane (cutout.cuh) runs the same code on real power rows.
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

__device__ __forceinline__ void cp_async4z(void* smem_dst, const void* gmem_src, bool valid) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  const int n = valid ? 4 : 0;  // 0: zero-fill, nothing is read
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(d), "l"(gmem_src), "r"(n) : "memory");
}
__device__ __forceinline__ void cp_async_elem(float2* d, const float2* s, bool valid) { cp_async8(d, s, valid); }
__device__ __forceinline__ void cp_async_elem(float* d, const float* s, bool valid) { cp_async4z(d, s, valid); }
__device__ __forceinline__ float inc_power(float2 v) { return __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y)); }
__device__ __forceinline__ float inc_power(float v) { return v; }

// One time tile [t0, t0 + INC_TILE) of a group of cnt <= INC_GROUP trials: acc[i][r] = sum over the C rows, in index
// order, of the row's power at t0 + lane + 32 r + the offset of trial warp + 16 i. Rows describes the rows:
//   raw_t                    float2 (a complex64 spectrum: the power is formed once per staged sample) or float (a
//                            power row, staged as it is)
//   row(c), len              row c, whose elements [0, len) are data; past len is read as 0
//   span(c)                  (min, max) of the group's offsets in row c
//   offsets(c, dst, tid, cnt) stores the group's offsets in row c to dst[0, cnt) (cp.async or plain shared stores; a
//                            barrier follows before they are read)
// smem: [INC_STAGES][span_max] raw_t, [span_max] float, [INC_STAGES][INC_GROUP] int (incoherent_smem_bytes for float2).
// The incoherent search (below) and the cut-outs' DM-time plane (cutout.cuh) both accumulate through here.
template <class Rows>
__device__ __forceinline__ void inc_tile(const Rows& rows, size_t C, size_t t0, int cnt, unsigned span_max,
                                         unsigned char* smem, float (&acc)[4][8]) {
  using raw_t = typename Rows::raw_t;
  raw_t* raw = reinterpret_cast<raw_t*>(smem);                               // [INC_STAGES][span_max]
  float* pw = reinterpret_cast<float*>(raw + INC_STAGES * (size_t)span_max);  // [span_max]
  int* s_off = reinterpret_cast<int*>(pw + span_max);                        // [INC_STAGES][INC_GROUP]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  // row c's span -> raw[c % 3], its offsets -> s_off[c % 3]; one commit group per row. The previous tile read raw and
  // s_off only before its last row's second barrier, so restaging them here is safe
  auto stage = [&](size_t c) {
    const int2 mm = rows.span(c);
    const size_t span = INC_TILE + (size_t)(mm.y - mm.x);
    const raw_t* row = rows.row(c);
    const size_t src0 = t0 + (size_t)mm.x;
    raw_t* dst = raw + (c % INC_STAGES) * (size_t)span_max;
    for (size_t e = tid; e < span; e += INC_THREADS) {
      const bool valid = src0 + e < rows.len;
      cp_async_elem(dst + e, valid ? row + src0 + e : row, valid);
    }
    rows.offsets(c, s_off + (c % INC_STAGES) * INC_GROUP, tid, cnt);
    cp_async_commit();
  };

#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int r = 0; r < 8; r++) acc[i][r] = 0.f;

  stage(0);
  if (C > 1) stage(1);
  else cp_async_commit();
  for (size_t c = 0; c < C; c++) {
    if (c + 2 < C) stage(c + 2);
    else cp_async_commit();  // empty groups keep wait_group 2 meaning "row c has landed"
    cp_async_wait2();
    __syncthreads();  // row c visible to all; every warp is done with the previous row's (or tile's) pw
    const int2 mm = rows.span(c);
    const size_t span = INC_TILE + (size_t)(mm.y - mm.x);
    const raw_t* src = raw + (c % INC_STAGES) * (size_t)span_max;
    for (size_t e = tid; e < span; e += INC_THREADS) pw[e] = inc_power(src[e]);
    // this row's offsets are read before the barrier: the next iteration's stage() overwrites s_off[c % 3]
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
}

// the incoherent search's rows: channel c of x, the group's offsets s + S- from the [C][n_dm] table
struct inc_spectrum_rows {
  using raw_t = float2;
  const float2* x;
  size_t len;  // L
  size_t n_dm;
  const int* goff;   // the group's first sorted slot of off
  const int2* gsp;   // the group's [C] spans
  __device__ __forceinline__ const float2* row(size_t c) const { return x + c * len; }
  __device__ __forceinline__ int2 span(size_t c) const { return gsp[c]; }
  __device__ __forceinline__ void offsets(size_t c, int* dst, int tid, int cnt) const {
    if (tid < cnt) cp_async4(dst + tid, goff + c * n_dm + tid);
  }
};

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
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t g = blockIdx.x;
  const int2 gi = groups[g];
  const int cnt = gi.y;
  const inc_spectrum_rows rows{x, L, n_dm, off + gi.x, gspan + g * C};
  const size_t tiles = (T + INC_TILE - 1) / INC_TILE;

  for (size_t tile = blockIdx.y; tile < tiles; tile += gridDim.y) {  // CTA-uniform
    const size_t t0 = tile * INC_TILE;
    float acc[4][8];
    inc_tile(rows, C, t0, cnt, span_max, inc_smem, acc);
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
