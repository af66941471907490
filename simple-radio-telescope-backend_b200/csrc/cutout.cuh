// cutout.cuh — per-candidate cut-outs of coherently dedispersed spectra (srtb_b200_candidate_cutouts): the dedispersed
// frequency-time image and the DM-time plane of each request, as include/srtb_b200.h defines them. Four launches per
// call whatever the number of requests, streams and rows:
//
//   cutout_plan_kernel      per request: the row DMs, and per channel the window base (the smallest shift any row or
//                           the image uses), the image's offset and each row group's (min, max) offset
//   cutout_decimate_kernel  per request and channel: the decimated power D(c, base_c + m), m < Wd, summed over the
//                           streams and q samples in order; only samples inside [0, ts) of kept channels are read
//   cutout_ft_kernel        the frequency-time image: subbands of D at the request's own DM
//   cutout_plane_kernel     the DM-time plane through the incoherent search's tile (incoherent.cuh: inc_tile) on the
//                           power rows D, a CTA per (request, group of <= 64 rows, 256 time bins); each row's shift is
//                           computed on the device as the row's offsets are staged
//
// Every sum is fp32 in the definition's order (streams, then samples, then channels), so two calls agree bit for bit.
#pragma once
#include <cuda_runtime.h>

#include "incoherent.cuh"

namespace srtb_b200 {

constexpr int CUT_THREADS = 256;

// one request as the kernels read it: t0 = center - (W/2) q
struct cut_request {
  long long t0;
  unsigned q;
  float dm, halfwidth;
};

// row r's DM: (float)(dm_req + halfwidth (r - n_rows/2) / (n_rows/2)), dm_req itself for a single row
__host__ __device__ inline float cut_row_dm(float dm_req, float halfwidth, unsigned r, unsigned n_rows) {
  if (n_rows == 1) return dm_req;
  const int h = (int)(n_rows / 2);
  return (float)((double)dm_req + (double)halfwidth * (double)((int)r - h) / (double)h);
}

// the shift of DM delta in decimated bins: llround(((delta - dm) k) / q), double, rounded half away from zero
__host__ __device__ inline long long cut_shift(float delta, double dm, double k, unsigned q) {
  return llround(((double)delta - dm) * k / (double)q);
}

// the spectra of one call: S streams of [C][L] complex64, data in [0, ts)
struct cut_spectra {
  const float2* x[4];
  int streams;
  size_t L, C, ts;
};

// grid (ceil(max(C, n_rows) / 256), n). row_dms [n][n_rows]; base, ft_off [n][C]; gspan [n][groups][C]
__global__ void __launch_bounds__(CUT_THREADS) cutout_plan_kernel(const cut_request* __restrict__ req,
                                                                  const double* __restrict__ k, size_t C, double dm,
                                                                  unsigned n_rows, unsigned rows_per_group,
                                                                  unsigned groups, float* __restrict__ row_dms,
                                                                  int* __restrict__ base, int* __restrict__ ft_off,
                                                                  int2* __restrict__ gspan) {
  const size_t n = blockIdx.y;
  const size_t t = (size_t)blockIdx.x * CUT_THREADS + threadIdx.x;
  const cut_request r = req[n];
  if (t < n_rows) row_dms[n * n_rows + t] = cut_row_dm(r.dm, r.halfwidth, (unsigned)t, n_rows);
  if (t >= C) return;
  const double kc = k[t];
  // DM_r is monotone in r and the shift in DM, so a run of rows spans the shifts of its end rows
  auto shift = [&](unsigned row) { return cut_shift(cut_row_dm(r.dm, r.halfwidth, row, n_rows), dm, kc, r.q); };
  const long long s_req = cut_shift(r.dm, dm, kc, r.q), s_first = shift(0), s_last = shift(n_rows - 1);
  const long long b = min(s_req, min(s_first, s_last));
  base[n * C + t] = (int)b;
  ft_off[n * C + t] = (int)(s_req - b);
  for (unsigned g = 0; g < groups; g++) {
    const unsigned r0 = g * rows_per_group, r1 = min(r0 + rows_per_group, n_rows) - 1;
    const long long a = shift(r0) - b, e = shift(r1) - b;
    gspan[(n * groups + g) * C + t] = make_int2((int)min(a, e), (int)max(a, e));
  }
}

// D [n][C][Wd]: D(c, base_c + m) = sum_{u < q} P(c, t0 + (base_c + m) q + u), P the stream-summed power of a kept
// channel inside [0, ts), else 0. A sample outside adds 0, which leaves the sum's bits as they are, so only the samples
// inside are read. Grid (C * tiles, n), tiles = ceil(Wd / 256): thread m of its channel's row.
__global__ void __launch_bounds__(CUT_THREADS) cutout_decimate_kernel(cut_spectra sp, const cut_request* __restrict__ req,
                                                                      const int* __restrict__ base, size_t Wd,
                                                                      unsigned tiles, float* __restrict__ D) {
  const size_t n = blockIdx.y;
  const size_t c = blockIdx.x / tiles;
  const size_t m = (size_t)(blockIdx.x % tiles) * CUT_THREADS + threadIdx.x;
  if (m >= Wd) return;
  bool kept = true;
#pragma unroll
  for (int s = 0; s < 4; s++)
    if (s < sp.streams) kept = kept && inc_power(sp.x[s][c * sp.L]) != 0.f;
  float acc = 0.f;
  if (kept) {
    const cut_request r = req[n];
    const long long q = r.q;
    const long long j0 = r.t0 + ((long long)base[n * sp.C + c] + (long long)m) * q;
    const long long lo = max(j0, 0ll), hi = min(j0 + q, (long long)sp.ts);
    const size_t row = c * sp.L;
    for (long long j = lo; j < hi; j++) {
      float p = inc_power(__ldg(sp.x[0] + row + j));
#pragma unroll
      for (int s = 1; s < 4; s++)
        if (s < sp.streams) p = __fadd_rn(p, inc_power(__ldg(sp.x[s] + row + j)));
      acc = __fadd_rn(acc, p);
    }
  }
  D[(n * sp.C + c) * Wd + m] = acc;
}

// ft [n][nsub][W]: subband k adds channels k C/nsub .. (k + 1) C/nsub - 1 in order. Grid (nsub * tiles, n)
__global__ void __launch_bounds__(CUT_THREADS) cutout_ft_kernel(const float* __restrict__ D,
                                                                const int* __restrict__ ft_off, size_t C, size_t Wd,
                                                                unsigned W, unsigned nsub, unsigned tiles,
                                                                float* __restrict__ ft) {
  const size_t n = blockIdx.y;
  const size_t k = blockIdx.x / tiles;
  const size_t i = (size_t)(blockIdx.x % tiles) * CUT_THREADS + threadIdx.x;
  if (i >= W) return;
  const size_t per = C / nsub;
  float acc = 0.f;
  for (size_t c = k * per; c < (k + 1) * per; c++) acc = __fadd_rn(acc, D[(n * C + c) * Wd + i + ft_off[n * C + c]]);
  ft[(n * nsub + k) * W + i] = acc;
}

// the plane's rows for inc_tile: channel c's power row D, each row's offset s(DM_r, c) - base_c computed as it is
// staged (plain shared stores; inc_tile's barrier follows)
struct cut_power_rows {
  using raw_t = float;
  const float* d;  // the request's [C][len]
  size_t len;      // Wd
  const int2* gsp;   // the group's [C] spans
  const int* base;   // the request's [C]
  const double* k;   // [C]
  const float* dms;  // the group's row DMs
  double dm;
  unsigned q;
  __device__ __forceinline__ const float* row(size_t c) const { return d + c * len; }
  __device__ __forceinline__ int2 span(size_t c) const { return gsp[c]; }
  __device__ __forceinline__ void offsets(size_t c, int* dst, int tid, int cnt) const {
    if (tid < cnt) dst[tid] = (int)(cut_shift(dms[tid], dm, k[c], q) - base[c]);
  }
};

// dmt [n][n_rows][W]. Grid (groups * tiles, n), tiles = ceil(W / INC_TILE); smem: inc_tile's for raw_t = float
__host__ __device__ constexpr size_t cutout_plane_smem_bytes(unsigned spread) {
  return (size_t)(INC_TILE + spread) * (INC_STAGES * sizeof(float) + sizeof(float)) + INC_STAGES * INC_GROUP * sizeof(int);
}
__global__ void __launch_bounds__(INC_THREADS) cutout_plane_kernel(
    const float* __restrict__ D, size_t C, size_t Wd, const int2* __restrict__ gspan, const int* __restrict__ base,
    const double* __restrict__ k, const float* __restrict__ row_dms, const cut_request* __restrict__ req, double dm,
    unsigned n_rows, unsigned rows_per_group, unsigned groups, unsigned W, unsigned span_max, float* __restrict__ dmt) {
  extern __shared__ __align__(16) unsigned char cut_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t n = blockIdx.y;
  const unsigned g = blockIdx.x % groups;
  const size_t t0 = (size_t)(blockIdx.x / groups) * INC_TILE;
  const unsigned r0 = g * rows_per_group;
  const int cnt = (int)min(rows_per_group, n_rows - r0);
  const cut_power_rows rows{D + n * C * Wd, Wd, gspan + (n * groups + g) * C, base + n * C, k,
                            row_dms + n * n_rows + r0, dm, req[n].q};
  float acc[4][8];
  inc_tile(rows, C, t0, cnt, span_max, cut_smem, acc);
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int kk = warp + 16 * i;
    if (kk >= cnt) continue;
    float* o = dmt + (n * n_rows + r0 + kk) * W;
#pragma unroll
    for (int r = 0; r < 8; r++) {
      const size_t j = t0 + lane + 32 * r;
      if (j < W) o[j] = acc[i][r];
    }
  }
}

}  // namespace srtb_b200
