// fold.cuh — fold 1 to 4 streams' dynamic spectra at a pulsar period into phase bins (srtb_b200_fold).
//
// Input per stream: x_s[C][L] complex64 (time contiguous), coherently dedispersed at `dm`. Sample j < F (fold_count)
// falls in phase bin bin(j) (fold_bin below; one formula for the device and the numpy restatement), and the call returns
//
//   profile[s][k][bin] = sum over the channels c of subband k and the j in bin of |x_s[c][j]|^2   (float64)
//   hits[bin]          = the number of j in bin
//   kept[s][k]         = the channels c of subband k with |x_s[c][0]|^2 != 0
//
// Three kernels, every sum in a fixed order (no float atomics: two calls agree bit for bit):
//
//   fold_plan_kernel     one CTA per time tile of FOLD_TILE samples: each j's bin, computed once; the tile's
//                        (bin, j) keys sorted (bitonic, keys unique), so a bin's samples are one contiguous run of the
//                        tile's sorted order. Writes the sorted (bin << 16 | j - tile start) list and adds the runs'
//                        lengths to hits (integer atomics).
//   fold_kernel          a CTA owns G channels of one subband of one stream and a range of tiles. Per tile every thread
//                        adds its FOLD_PER_THREAD samples' |x|^2 over the G channels in channel order (float64; so the
//                        spectrum is read once and the binning below runs once per G channels), then the tile's sorted
//                        order is cut into equal chunks, one per thread: a bin whose run lies inside one chunk is added
//                        by that thread, a run that crosses chunks by the thread holding its start, which walks the
//                        following chunks' carries in order. acc[bin] lives in shared memory for the CTA's tiles and is
//                        stored once: one float64 row of nbin per CTA.
//   fold_finish_kernel   adds each output's CTA rows (channel groups, then tile ranges, in index order) and the groups'
//                        kept counts. Not launched when every subband has one CTA: fold_kernel then stores the output.
//
// fold_coherence_kernel (srtb_b200_fold_coherence) takes fold_kernel's place for a stream pair: the coherence products
// AA, BB, CR, CI of X = x_0 and Y = x_1 over the channels kept in both, between the same plan and finish kernels.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace srtb_b200 {

constexpr int FOLD_TILE = 2048;          // time samples per tile (sorted as one list)
constexpr int FOLD_THREADS = 256;        // fold_kernel
constexpr int FOLD_PER_THREAD = FOLD_TILE / FOLD_THREADS;
constexpr int FOLD_PLAN_THREADS = 1024;  // fold_plan_kernel: two keys per thread
constexpr int FOLD_MAX_BINS = 4096;      // bin fits 13 bits; the sentinel bin nbin marks j >= F
constexpr int FOLD_MAX_GROUP = 64;       // channels per fold_kernel CTA, at most

struct fold_spectra {
  const float2* x[4];
};

// the bin of sample j: p = (phi0 + a j) + b (j j), f = p - floor(p), bin = min(floor(f nbin), nbin - 1), each operation
// rounded on its own (no FMA contraction), so numpy's float64 arithmetic reproduces it
__device__ __forceinline__ int fold_bin(double phi0, double a, double b, int nbin, long long j) {
  const double jd = (double)j;
  const double p = __dadd_rn(__dadd_rn(phi0, __dmul_rn(a, jd)), __dmul_rn(b, __dmul_rn(jd, jd)));
  const double f = __dsub_rn(p, floor(p));
  const int bin = (int)floor(__dmul_rn(f, (double)nbin));
  return bin < nbin - 1 ? bin : nbin - 1;
}

// grid: one CTA per tile. plan[tile][FOLD_TILE]: sorted bin << 16 | local j; samples j >= F carry the bin nbin
__global__ void __launch_bounds__(FOLD_PLAN_THREADS) fold_plan_kernel(double phi0, double a, double b, int nbin,
                                                                      long long F, uint32_t* __restrict__ plan,
                                                                      unsigned long long* __restrict__ hits) {
  __shared__ uint32_t key[FOLD_TILE];
  const long long j0 = (long long)blockIdx.x * FOLD_TILE;
  for (int i = threadIdx.x; i < FOLD_TILE; i += FOLD_PLAN_THREADS) {
    const long long j = j0 + i;
    const int bin = j < F ? fold_bin(phi0, a, b, nbin, j) : nbin;
    key[i] = ((uint32_t)bin << 16) | (uint32_t)i;
  }
  __syncthreads();
  for (int k = 2; k <= FOLD_TILE; k <<= 1)
    for (int m = k >> 1; m > 0; m >>= 1) {
      for (int i = threadIdx.x; i < FOLD_TILE; i += FOLD_PLAN_THREADS) {
        const int l = i ^ m;
        if (l > i) {
          const uint32_t u = key[i], v = key[l];
          const bool up = (i & k) == 0;
          if ((u > v) == up) {
            key[i] = v;
            key[l] = u;
          }
        }
      }
      __syncthreads();
    }
  uint32_t* out = plan + (size_t)blockIdx.x * FOLD_TILE;
  for (int i = threadIdx.x; i < FOLD_TILE; i += FOLD_PLAN_THREADS) {
    const uint32_t k = key[i];
    out[i] = k;
    const uint32_t bin = k >> 16;
    if (bin >= (uint32_t)nbin) continue;
    if (i > 0 && (key[i - 1] >> 16) == bin) continue;  // not the start of its bin's run
    int e = i + 1;
    while (e < FOLD_TILE && (key[e] >> 16) == bin) e++;
    atomicAdd(hits + bin, (unsigned long long)(e - i));
  }
}

// dynamic shared memory of fold_kernel
__host__ __device__ constexpr size_t fold_smem_bytes(int nbin) {
  return (size_t)(nbin + 1) * sizeof(double) + FOLD_TILE * sizeof(double) + FOLD_THREADS * (sizeof(double) + sizeof(int));
}

// grid.x = streams * C / G (stream-major channel groups), grid.y = tile ranges. out row of CTA (s, group g, range r):
// ((s * C / G + g) * gridDim.y + r) * nbin; kept_out[s * C / G + g] from the CTAs of range 0
__global__ void __launch_bounds__(FOLD_THREADS, 4) fold_kernel(fold_spectra sp, size_t L, int C, int G, int nbin,
                                                            long long F, int ntiles, const uint32_t* __restrict__ plan,
                                                            double* __restrict__ out, unsigned* __restrict__ kept_out) {
  extern __shared__ double smem[];
  double* acc = smem;                               // [nbin + 1]: the last one takes the padding samples
  double* pw = acc + nbin + 1;                      // [FOLD_TILE]: summed power by local j
  double* carry = pw + FOLD_TILE;                   // [FOLD_THREADS]: a chunk's sum before its first run start
  int* has_start = reinterpret_cast<int*>(carry + FOLD_THREADS);
  const int groups = C / G;
  const int s = blockIdx.x / groups, g = blockIdx.x % groups;
  // selected, not indexed: a parameter array indexed at run time is copied to the stack
  const float2* xs = s == 0 ? sp.x[0] : s == 1 ? sp.x[1] : s == 2 ? sp.x[2] : sp.x[3];
  const float2* x = xs + (size_t)g * G * L;
  const int t = threadIdx.x;
  for (int i = t; i <= nbin; i += FOLD_THREADS) acc[i] = 0.0;
  const int r = blockIdx.y, R = gridDim.y;
  const int tile_lo = (int)((long long)ntiles * r / R), tile_hi = (int)((long long)ntiles * (r + 1) / R);
  unsigned kept = 0;
  for (int tile = tile_lo; tile < tile_hi; tile++) {
    const long long j0 = (long long)tile * FOLD_TILE;
    double v[FOLD_PER_THREAD];
#pragma unroll
    for (int e = 0; e < FOLD_PER_THREAD; e++) v[e] = 0.0;
    for (int c = 0; c < G; c++) {
      const float2* row = x + (size_t)c * L;
      float2 q[FOLD_PER_THREAD];
#pragma unroll
      for (int e = 0; e < FOLD_PER_THREAD; e++) {
        const long long j = j0 + t + e * FOLD_THREADS;
        q[e] = j < F ? __ldcs(row + j) : make_float2(0.f, 0.f);
      }
#pragma unroll
      for (int e = 0; e < FOLD_PER_THREAD; e++)  // |x|^2 in fp32 (relative error 2^-23), added in float64
        v[e] = __dadd_rn(v[e], (double)__fadd_rn(__fmul_rn(q[e].x, q[e].x), __fmul_rn(q[e].y, q[e].y)));
      if (tile == 0 && t == 0) kept += (q[0].x * q[0].x + q[0].y * q[0].y != 0.f) ? 1u : 0u;  // the detector's rule
    }
#pragma unroll
    for (int e = 0; e < FOLD_PER_THREAD; e++) pw[t + e * FOLD_THREADS] = v[e];
    __syncthreads();
    // this thread's chunk of the sorted order: complete runs go straight to acc, the rest to carry / tail
    const uint32_t* pl = plan + (size_t)tile * FOLD_TILE + t * FOLD_PER_THREAD;
    uint32_t prev_bin = t > 0 ? (pl[-1] >> 16) : 0xffffffffu;
    bool started = false;
    double cur = 0.0;
    uint32_t cur_bin = 0;
#pragma unroll
    for (int e = 0; e < FOLD_PER_THREAD; e++) {
      const uint32_t k = pl[e], bin = k >> 16;
      if (bin != prev_bin) {
        if (started) acc[cur_bin] = __dadd_rn(acc[cur_bin], cur);
        else carry[t] = cur;
        started = true;
        cur = 0.0;
        cur_bin = bin;
        prev_bin = bin;
      }
      cur = __dadd_rn(cur, pw[k & 0xffffu]);
    }
    if (!started) carry[t] = cur;
    has_start[t] = started ? 1 : 0;
    __syncthreads();
    if (started) {  // the last run started here: add the following chunks' carries up to the next run start
      for (int u = t + 1; u < FOLD_THREADS; u++) {
        cur = __dadd_rn(cur, carry[u]);
        if (has_start[u]) break;
      }
      acc[cur_bin] = __dadd_rn(acc[cur_bin], cur);
    }
    __syncthreads();
  }
  double* o = out + (size_t)(blockIdx.x * (size_t)R + r) * nbin;
  for (int i = t; i < nbin; i += FOLD_THREADS) o[i] = acc[i];
  if (r == 0 && t == 0) kept_out[blockIdx.x] = kept;
}

// ---- coherence products of a stream pair (srtb_b200_fold_coherence): X = x_0, Y = x_1 and, for the channels c kept in
// both (|X[c][0]|^2 != 0 and |Y[c][0]|^2 != 0, in fp32 as fold_kernel's rule), the four sums
//   AA = |X|^2, BB = |Y|^2, CR = Re(X conj Y), CI = Im(X conj Y)
// over the channels of subband k and the j in bin. The bin plan is fold_plan_kernel's and the CTA rows are added by
// fold_finish_kernel, with the four products in the place of the streams. Every product of two fp32 components is exact
// in float64, so CR and CI, which cancel heavily on unpolarised noise, carry only the float64 rounding of their sums.
constexpr int FOLD_COH_THREADS = 256;  // fold_coherence_kernel
constexpr int FOLD_COH_PER_THREAD = FOLD_TILE / FOLD_COH_THREADS;

// dynamic shared memory of fold_coherence_kernel: acc [nbin + 1][4], pw [FOLD_TILE][4], carry [threads][4], has_start
__host__ __device__ constexpr size_t fold_coherence_smem_bytes(int nbin) {
  return (size_t)(nbin + 1) * 4 * sizeof(double) + FOLD_TILE * 4 * sizeof(double) +
         FOLD_COH_THREADS * (4 * sizeof(double) + sizeof(int));
}

// grid.x = C / G channel groups, grid.y = tile ranges. out row of CTA (product p, group g, range r):
// ((p * C / G + g) * gridDim.y + r) * nbin; kept_out[p * C / G + g] (the same count for each p, from the CTAs of range
// 0), so fold_finish_kernel adds rows and counts for 4 "streams". A channel masked in either stream is skipped: its
// samples are not loaded and it adds nothing to any product
__global__ void __launch_bounds__(FOLD_COH_THREADS, 2) fold_coherence_kernel(
    const float2* __restrict__ xs, const float2* __restrict__ ys, size_t L, int C, int G, int nbin, long long F,
    int ntiles, const uint32_t* __restrict__ plan, double* __restrict__ out, unsigned* __restrict__ kept_out) {
  extern __shared__ double smem[];
  double* acc = smem;                                     // [nbin + 1][4]: the last bin takes the padding samples
  double* pw = acc + (size_t)(nbin + 1) * 4;              // [FOLD_TILE][4]: the summed products by local j
  double* carry = pw + FOLD_TILE * 4;                     // [threads][4]: a chunk's sums before its first run start
  int* has_start = reinterpret_cast<int*>(carry + FOLD_COH_THREADS * 4);
  __shared__ uint32_t keep_bits[FOLD_MAX_GROUP / 32];
  const int groups = C / G, g = blockIdx.x;
  const float2* x = xs + (size_t)g * G * L;
  const float2* y = ys + (size_t)g * G * L;
  const int t = threadIdx.x;
  for (int i = t; i < (nbin + 1) * 4; i += FOLD_COH_THREADS) acc[i] = 0.0;
  if (t < FOLD_MAX_GROUP) {  // the pair's mask of the group's channels, one bit each
    bool keep = false;
    if (t < G) {
      const float2 a = x[(size_t)t * L], b = y[(size_t)t * L];
      keep = __fadd_rn(__fmul_rn(a.x, a.x), __fmul_rn(a.y, a.y)) != 0.f &&
             __fadd_rn(__fmul_rn(b.x, b.x), __fmul_rn(b.y, b.y)) != 0.f;
    }
    const uint32_t bits = __ballot_sync(0xffffffffu, keep);
    if ((t & 31) == 0) keep_bits[t >> 5] = bits;
  }
  __syncthreads();
  const int r = blockIdx.y, R = gridDim.y;
  const int tile_lo = (int)((long long)ntiles * r / R), tile_hi = (int)((long long)ntiles * (r + 1) / R);
  for (int tile = tile_lo; tile < tile_hi; tile++) {
    const long long j0 = (long long)tile * FOLD_TILE;
    double aa[FOLD_COH_PER_THREAD], bb[FOLD_COH_PER_THREAD], cr[FOLD_COH_PER_THREAD], ci[FOLD_COH_PER_THREAD];
#pragma unroll
    for (int e = 0; e < FOLD_COH_PER_THREAD; e++) aa[e] = bb[e] = cr[e] = ci[e] = 0.0;
    for (int c = 0; c < G; c++) {
      if (!((keep_bits[c >> 5] >> (c & 31)) & 1u)) continue;  // masked in X or Y: in no product
      const float2* xrow = x + (size_t)c * L;
      const float2* yrow = y + (size_t)c * L;
      float2 p[FOLD_COH_PER_THREAD], q[FOLD_COH_PER_THREAD];
#pragma unroll
      for (int e = 0; e < FOLD_COH_PER_THREAD; e++) {
        const long long j = j0 + t + e * FOLD_COH_THREADS;
        p[e] = j < F ? __ldcs(xrow + j) : make_float2(0.f, 0.f);
        q[e] = j < F ? __ldcs(yrow + j) : make_float2(0.f, 0.f);
      }
#pragma unroll
      for (int e = 0; e < FOLD_COH_PER_THREAD; e++) {  // each product exact in float64; one rounding per add
        const double xr = p[e].x, xi = p[e].y, yr = q[e].x, yi = q[e].y;
        aa[e] = __dadd_rn(aa[e], __dadd_rn(__dmul_rn(xr, xr), __dmul_rn(xi, xi)));
        bb[e] = __dadd_rn(bb[e], __dadd_rn(__dmul_rn(yr, yr), __dmul_rn(yi, yi)));
        cr[e] = __dadd_rn(cr[e], __dadd_rn(__dmul_rn(xr, yr), __dmul_rn(xi, yi)));
        ci[e] = __dadd_rn(ci[e], __dsub_rn(__dmul_rn(xi, yr), __dmul_rn(xr, yi)));
      }
    }
#pragma unroll
    for (int e = 0; e < FOLD_COH_PER_THREAD; e++) {
      double2* o = reinterpret_cast<double2*>(pw + (size_t)(t + e * FOLD_COH_THREADS) * 4);
      o[0] = make_double2(aa[e], bb[e]);
      o[1] = make_double2(cr[e], ci[e]);
    }
    __syncthreads();
    // this thread's chunk of the sorted order, as in fold_kernel, with four sums per run
    const uint32_t* pl = plan + (size_t)tile * FOLD_TILE + t * FOLD_COH_PER_THREAD;
    uint32_t prev_bin = t > 0 ? (pl[-1] >> 16) : 0xffffffffu;
    bool started = false;
    double2 c0 = make_double2(0.0, 0.0), c1 = c0;
    uint32_t cur_bin = 0;
#pragma unroll
    for (int e = 0; e < FOLD_COH_PER_THREAD; e++) {
      const uint32_t k = pl[e], bin = k >> 16;
      if (bin != prev_bin) {
        double2* dst = reinterpret_cast<double2*>(started ? acc + (size_t)cur_bin * 4 : carry + t * 4);
        if (started) {
          c0 = make_double2(__dadd_rn(dst[0].x, c0.x), __dadd_rn(dst[0].y, c0.y));
          c1 = make_double2(__dadd_rn(dst[1].x, c1.x), __dadd_rn(dst[1].y, c1.y));
        }
        dst[0] = c0;
        dst[1] = c1;
        started = true;
        c0 = c1 = make_double2(0.0, 0.0);
        cur_bin = bin;
        prev_bin = bin;
      }
      const double2* src = reinterpret_cast<const double2*>(pw + (size_t)(k & 0xffffu) * 4);
      const double2 s0 = src[0], s1 = src[1];
      c0 = make_double2(__dadd_rn(c0.x, s0.x), __dadd_rn(c0.y, s0.y));
      c1 = make_double2(__dadd_rn(c1.x, s1.x), __dadd_rn(c1.y, s1.y));
    }
    if (!started) {
      double2* dst = reinterpret_cast<double2*>(carry + t * 4);
      dst[0] = c0;
      dst[1] = c1;
    }
    has_start[t] = started ? 1 : 0;
    __syncthreads();
    if (started) {  // the last run started here: add the following chunks' carries up to the next run start
      for (int u = t + 1; u < FOLD_COH_THREADS; u++) {
        const double2* cu = reinterpret_cast<const double2*>(carry + u * 4);
        c0 = make_double2(__dadd_rn(c0.x, cu[0].x), __dadd_rn(c0.y, cu[0].y));
        c1 = make_double2(__dadd_rn(c1.x, cu[1].x), __dadd_rn(c1.y, cu[1].y));
        if (has_start[u]) break;
      }
      double2* dst = reinterpret_cast<double2*>(acc + (size_t)cur_bin * 4);
      dst[0] = make_double2(__dadd_rn(dst[0].x, c0.x), __dadd_rn(dst[0].y, c0.y));
      dst[1] = make_double2(__dadd_rn(dst[1].x, c1.x), __dadd_rn(dst[1].y, c1.y));
    }
    __syncthreads();
  }
  for (int p = 0; p < 4; p++) {
    double* o = out + ((size_t)(p * groups + g) * R + r) * nbin;
    for (int i = t; i < nbin; i += FOLD_COH_THREADS) o[i] = acc[(size_t)i * 4 + p];
  }
  if (r == 0 && t < 4) kept_out[t * groups + g] = __popc(keep_bits[0]) + __popc(keep_bits[1]);
}

// one thread per output (s, k, bin): adds the rows of its subband's groups and tile ranges in index order; the bin-0
// thread also adds the groups' kept counts
__global__ void __launch_bounds__(256) fold_finish_kernel(const double* __restrict__ rows,
                                                          const unsigned* __restrict__ kept_rows, int rows_per_output,
                                                          int groups_per_sub, int nbin, size_t outputs,
                                                          double* __restrict__ profile, unsigned* __restrict__ kept) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= outputs) return;
  const size_t sk = i / nbin, bin = i % nbin;
  const double* r = rows + sk * rows_per_output * (size_t)nbin + bin;
  double acc = 0.0;
  for (int q = 0; q < rows_per_output; q++) acc = __dadd_rn(acc, r[(size_t)q * nbin]);
  profile[i] = acc;
  if (bin == 0) {
    unsigned n = 0;
    for (int q = 0; q < groups_per_sub; q++) n += kept_rows[sk * groups_per_sub + q];
    kept[sk] = n;
  }
}

}  // namespace srtb_b200
