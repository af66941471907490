// fft_engine.cuh — hand-written sm_90a FFT passes (no cuFFT on the hot path).
//
// Replaces the vendor-FFT call sites of the reference:
//   R2C  : userspace/include/srtb/fft/cufft_like_wrapper.hpp:183-191 (cufftExecR2C)
//   C2C  : userspace/include/srtb/fft/cufft_like_wrapper.hpp:205-207 (batched, waterfall)
// and the in-tree fallback userspace/include/srtb/fft/naive_fft.hpp:155-176,221-261,
// whose transform definition (unnormalised, forward = e^{-2 pi i nk/N}) is kept.
//
// One kernel template implements one "pass": a Stockham auto-sort FFT of length
// L = 2^LOGL on a tile of T independent sequences held in shared memory, eight points
// per thread per stage in registers (radix 8/4/2 butterflies), the first stage loading
// straight from HBM and the last stage storing straight to HBM.
//   MODE_ROW   : sequences are contiguous rows (lanes run along the FFT index)
//   MODE_COL   : sequences are strided columns, T neighbours contiguous (lanes run along T)
//   MODE_TRANS : loads like ROW, stores like COL (the transposing last pass of a
//                multi-pass transform, which produces natural order)
// A length-n transform with n > 4096 is n = L1*L2(*L3): COL pass(es) with the inter-pass
// twiddle fused into the store, then one TRANS pass (see fft_plan in srtb_b200_fft.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace srtb_b200 {

enum { MODE_ROW = 0, MODE_COL = 1, MODE_TRANS = 2 };

__device__ __forceinline__ float2 c_add(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 c_sub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 c_mul(float2 a, float2 b) {
  return make_float2(fmaf(a.x, b.x, -a.y * b.y), fmaf(a.x, b.y, a.y * b.x));
}
__device__ __forceinline__ float2 c_sqr(float2 a) {
  return make_float2(fmaf(a.x, a.x, -a.y * a.y), 2.0f * a.x * a.y);
}
// multiply by -i (forward) / +i (backward)
template <bool FWD>
__device__ __forceinline__ float2 c_rot(float2 a) {
  return FWD ? make_float2(a.y, -a.x) : make_float2(-a.y, a.x);
}
template <bool FWD>
__device__ __forceinline__ float2 c_dir(float2 w) {  // table holds forward twiddles
  return FWD ? w : make_float2(w.x, -w.y);
}

// ---- in-register DFTs, natural-order in and out -----------------------------------
template <bool FWD>
__device__ __forceinline__ void dft2(float2& a, float2& b) {
  const float2 t = a;
  a = c_add(t, b);
  b = c_sub(t, b);
}
template <bool FWD>
__device__ __forceinline__ void dft4(float2& a0, float2& a1, float2& a2, float2& a3) {
  const float2 t0 = c_add(a0, a2), t1 = c_sub(a0, a2);
  const float2 t2 = c_add(a1, a3), t3 = c_rot<FWD>(c_sub(a1, a3));
  a0 = c_add(t0, t2);
  a1 = c_add(t1, t3);
  a2 = c_sub(t0, t2);
  a3 = c_sub(t1, t3);
}
template <bool FWD>
__device__ __forceinline__ void dft8(float2& v0, float2& v1, float2& v2, float2& v3, float2& v4,
                                     float2& v5, float2& v6, float2& v7) {
  dft4<FWD>(v0, v2, v4, v6);  // E0..E3 in v0,v2,v4,v6
  dft4<FWD>(v1, v3, v5, v7);  // O0..O3 in v1,v3,v5,v7
  constexpr float c = 0.70710678118654752440f;
  // O1 *= W8^1, O2 *= W8^2, O3 *= W8^3
  const float2 o1 = FWD ? make_float2(c * (v3.x + v3.y), c * (v3.y - v3.x))
                        : make_float2(c * (v3.x - v3.y), c * (v3.x + v3.y));
  const float2 o2 = c_rot<FWD>(v5);
  const float2 o3 = FWD ? make_float2(c * (v7.y - v7.x), -c * (v7.x + v7.y))
                        : make_float2(-c * (v7.x + v7.y), c * (v7.x - v7.y));
  const float2 e0 = v0, e1 = v2, e2 = v4, e3 = v6, o0 = v1;
  v0 = c_add(e0, o0);
  v4 = c_sub(e0, o0);
  v1 = c_add(e1, o1);
  v5 = c_sub(e1, o1);
  v2 = c_add(e2, o2);
  v6 = c_sub(e2, o2);
  v3 = c_add(e3, o3);
  v7 = c_sub(e3, o3);
}

// ---- stage schedule: radix-8 stages first, remainder (radix 4 or 2) last ------------
template <int LOGL>
struct sched {
  static constexpr int S = (LOGL + 2) / 3;
  __host__ __device__ static constexpr int logr(int s) { return (s < S - 1) ? 3 : (LOGL - 3 * (S - 1)); }
  __host__ __device__ static constexpr int logns(int s) { return 3 * s; }  // all stages before s are radix 8
};

// One Stockham stage on the eight values a thread holds.
// Slot e of v[] is the point read at index u + e*U (U = L/8). A radix-r stage treats the
// slots as NB = 8/r butterflies: butterfly m uses slots m + i*NB (i < r) and is butterfly
// number u + m*U of the L/r butterflies in the sequence. Twiddle (DIT) W_{Ns*r}^{k*i},
// k = butterfly % Ns; outputs go to (b / Ns)*Ns*r + k + i*Ns.
// TABLE = true reads every power W^{k i} from the table (cheap when the lanes of a warp share k, i.e.
// in the column-mode mappings); TABLE = false reads W^k and forms the powers by multiplication
// (lanes run along k: one gather instead of seven).
// TWSHIFT: table index of W_{Ns*R}^j is j << TWSHIFT (LOGL - LOGNS - LOGR for a length-L table, 0 for
// a per-stage compact table). TWLDG: the table is in global memory (read through the read-only path)
// rather than in shared memory.
template <int LOGL, int LOGR, int LOGNS, bool FWD, bool TABLE = false, int TWSHIFT = LOGL - LOGNS - LOGR,
          bool TWLDG = true>
__device__ __forceinline__ void stage_compute(float2 (&v)[8], int u, const float2* __restrict__ tw,
                                              int (&oidx)[8]) {
  constexpr int L = 1 << LOGL, U = L / 8, R = 1 << LOGR, NB = 8 / R, NS = 1 << LOGNS;
#pragma unroll
  for (int m = 0; m < NB; m++) {
    const int b = u + m * U;
    const int k = b & (NS - 1);
    if constexpr (LOGNS > 0) {
      // w1 = W_{Ns*R}^k from the length-L forward table; higher powers by multiplication
      constexpr int SH = (TWSHIFT < 0) ? 0 : TWSHIFT;
      const float2 w1 = c_dir<FWD>(TWLDG ? __ldg(&tw[k << SH]) : tw[k << SH]);
      if (R == 2) {
        v[m + NB] = c_mul(v[m + NB], w1);
      } else if (TABLE) {
#pragma unroll
        for (int i = 1; i < R; i++) {
          const float2 wi = (i == 1) ? w1 : c_dir<FWD>(TWLDG ? __ldg(&tw[(k * i) << SH]) : tw[(k * i) << SH]);
          v[m + i * NB] = c_mul(v[m + i * NB], wi);
        }
      } else if (R == 4) {
        const float2 w2 = c_sqr(w1), w3 = c_mul(w2, w1);
        v[m + NB] = c_mul(v[m + NB], w1);
        v[m + 2 * NB] = c_mul(v[m + 2 * NB], w2);
        v[m + 3 * NB] = c_mul(v[m + 3 * NB], w3);
      } else {
        const float2 w2 = c_sqr(w1), w3 = c_mul(w2, w1), w4 = c_sqr(w2);
        const float2 w5 = c_mul(w4, w1), w6 = c_sqr(w3), w7 = c_mul(w4, w3);
        v[m + 1] = c_mul(v[m + 1], w1);
        v[m + 2] = c_mul(v[m + 2], w2);
        v[m + 3] = c_mul(v[m + 3], w3);
        v[m + 4] = c_mul(v[m + 4], w4);
        v[m + 5] = c_mul(v[m + 5], w5);
        v[m + 6] = c_mul(v[m + 6], w6);
        v[m + 7] = c_mul(v[m + 7], w7);
      }
    }
    if (R == 2) {
      dft2<FWD>(v[m], v[m + NB]);
    } else if (R == 4) {
      dft4<FWD>(v[m], v[m + NB], v[m + 2 * NB], v[m + 3 * NB]);
    } else {
      dft8<FWD>(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7]);
    }
    const int obase = ((b >> LOGNS) << (LOGNS + LOGR)) + k;
#pragma unroll
    for (int i = 0; i < R; i++) oidx[m + i * NB] = obase + i * NS;
  }
}


// ---- sixteen points per thread (radix-16 stages): half the shared-memory round trips and barriers of
// the eight-point schedule for L = 256 (16 x 16) and L = 128 (16 x 8) ------------------------------
template <bool FWD>
__device__ __forceinline__ float2 c_mulc(float2 a, float wr, float wi_fwd) {  // a * (wr, wi), table holds forward
  const float wi = FWD ? wi_fwd : -wi_fwd;
  return make_float2(fmaf(a.x, wr, -a.y * wi), fmaf(a.x, wi, a.y * wr));
}
// multiply by W8^1 = (c, -c) and W8^3 = (-c, -c) (forward; conjugates backward)
template <bool FWD>
__device__ __forceinline__ float2 c_w8_1(float2 a) {
  constexpr float c = 0.70710678118654752440f;
  return FWD ? make_float2(c * (a.x + a.y), c * (a.y - a.x)) : make_float2(c * (a.x - a.y), c * (a.x + a.y));
}
template <bool FWD>
__device__ __forceinline__ float2 c_w8_3(float2 a) {
  constexpr float c = 0.70710678118654752440f;
  return FWD ? make_float2(c * (a.y - a.x), -c * (a.x + a.y)) : make_float2(-c * (a.x + a.y), c * (a.x - a.y));
}
template <bool FWD>
__device__ __forceinline__ void dft16(float2 (&a)[16]) {
  constexpr float C1 = 0.92387953251128675613f, S1 = 0.38268343236508977173f;
#pragma unroll
  for (int j = 0; j < 4; j++) dft4<FWD>(a[j], a[j + 4], a[j + 8], a[j + 12]);  // a[j + 4q] = A_j[q]
  // A_j[q] *= W16^{j q}
  a[5] = c_mulc<FWD>(a[5], C1, -S1);    // j=1,q=1: W^1
  a[9] = c_w8_1<FWD>(a[9]);             // j=1,q=2: W^2
  a[13] = c_mulc<FWD>(a[13], S1, -C1);  // j=1,q=3: W^3
  a[6] = c_w8_1<FWD>(a[6]);             // j=2,q=1: W^2
  a[10] = c_rot<FWD>(a[10]);            // j=2,q=2: W^4
  a[14] = c_w8_3<FWD>(a[14]);           // j=2,q=3: W^6
  a[7] = c_mulc<FWD>(a[7], S1, -C1);    // j=3,q=1: W^3
  a[11] = c_w8_3<FWD>(a[11]);           // j=3,q=2: W^6
  a[15] = c_mulc<FWD>(a[15], -C1, S1);  // j=3,q=3: W^9
#pragma unroll
  for (int q = 0; q < 4; q++) dft4<FWD>(a[4 * q], a[4 * q + 1], a[4 * q + 2], a[4 * q + 3]);  // a[4q+p] = X[q+4p]
#pragma unroll
  for (int q = 0; q < 4; q++)
#pragma unroll
    for (int p = q + 1; p < 4; p++) {
      const float2 tmp = a[4 * q + p];
      a[4 * q + p] = a[4 * p + q];
      a[4 * p + q] = tmp;
    }
}

template <int LOGL>
struct sched16 {
  // two stages up to L = 256 (16 x 2^(LOGL-4)); three above: 512 = 16*8*4, 1024 = 16*16*4, 2048 = 16*16*8,
  // 4096 = 16^3 (every radix is 4, 8 or 16)
  static constexpr int S = (LOGL <= 8) ? 2 : 3;
  __host__ __device__ static constexpr int logr(int s) {
    if (LOGL <= 8) return s == 0 ? 4 : LOGL - 4;
    if (LOGL == 9) return s == 0 ? 4 : (s == 1 ? 3 : 2);
    return s < 2 ? 4 : LOGL - 8;
  }
  __host__ __device__ static constexpr int logns(int s) {
    int a = 0;
    for (int i = 0; i < s; i++) a += logr(i);
    return a;
  }
};

// stage_compute for sixteen slots: slot e is the point read at u + e*U (U = L/16); radix 16 (one
// butterfly), 8 (two), 4 (four). Twiddles always come from the table (column-mode mapping).
// PAD: the output slots are returned for a tile whose rows carry one spare row after every sixteen
// (row r sits at r + (r >> 4)); with NS = 1 (radix 16 first) or NS a multiple of 16 this stays base + i * constant.
template <int LOGL, int LOGR, int LOGNS, bool FWD, int TWSHIFT = LOGL - LOGNS - LOGR, bool PAD = false>
__device__ __forceinline__ void stage_compute16(float2 (&v)[16], int u, const float2* __restrict__ tw,
                                                int (&oidx)[16]) {
  constexpr int L = 1 << LOGL, U = L / 16, R = 1 << LOGR, NB = 16 / R, NS = 1 << LOGNS;
  static_assert(LOGR >= 2 && LOGR <= 4, "radix 4, 8 or 16");
  static_assert(!PAD || NS >= 16 || (NS == 1 && LOGR == 4), "padded rows: slot stride must keep the pad linear");
#pragma unroll
  for (int m = 0; m < NB; m++) {
    const int b = u + m * U;
    const int k = b & (NS - 1);
    if constexpr (LOGNS > 0) {
      constexpr int SH = (TWSHIFT < 0) ? 0 : TWSHIFT;
#pragma unroll
      for (int i = 1; i < R; i++) v[m + i * NB] = c_mul(v[m + i * NB], c_dir<FWD>(tw[(k * i) << SH]));
    }
    if constexpr (R == 16) {
      dft16<FWD>(v);
    } else if constexpr (R == 8) {
      dft8<FWD>(v[m], v[m + 2], v[m + 4], v[m + 6], v[m + 8], v[m + 10], v[m + 12], v[m + 14]);
    } else {
      dft4<FWD>(v[m], v[m + 4], v[m + 8], v[m + 12]);
    }
    const int obase = ((b >> LOGNS) << (LOGNS + LOGR)) + k;
    if constexpr (PAD) {
      const int pbase = obase + (obase >> 4);
      constexpr int PSTEP = NS >= 16 ? NS + NS / 16 : NS;
#pragma unroll
      for (int i = 0; i < R; i++) oidx[m + i * NB] = pbase + i * PSTEP;
    } else {
#pragma unroll
      for (int i = 0; i < R; i++) oidx[m + i * NB] = obase + i * NS;
    }
  }
}

// shared-memory layout of the tile
template <int LOGL, int T, int MODE>
struct tile_layout {
  static constexpr int L = 1 << LOGL;
  static constexpr int LPAD = L + (L >> 4);
  static constexpr int ELEMS = (MODE == MODE_ROW) ? T * LPAD : T * L;
  __device__ __forceinline__ static int at(int idx, int t) {
    if (MODE == MODE_ROW) return t * LPAD + idx + (idx >> 4);
    if (MODE == MODE_COL) return idx * T + t;
    return idx * T + ((t + (idx >> 3)) & (T - 1));  // TRANS: rotate so both maps are conflict-free
  }
};

template <int LOGL, int T>
struct pass_threads {
  static constexpr int value = ((1 << LOGL) / 8) * T;
  // resident CTAs per SM the persistent TMA kernels aim for (register budget via __launch_bounds__)
  static constexpr int min_blocks = (value >= 1024) ? 1 : ((value >= 512) ? 3 : ((value >= 256) ? 5 : 8));
};

// IO concept:
//   bool  IO::tile_valid(int t)                     sequence t of this tile exists
//   float2 IO::load(int t, int pos)                  point `pos` of sequence t
//   void  IO::store8(int t, int u, int U, float2 (&v)[8])   outputs k = u + e*U, e = 0..7
template <int LOGL, int T, int MODE, bool FWD, class IO>
__global__ void __launch_bounds__(pass_threads<LOGL, T>::value)
    fft_pass_kernel(IO io, const float2* __restrict__ tw) {
  using SC = sched<LOGL>;
  using LAY = tile_layout<LOGL, T, MODE>;
  constexpr int L = 1 << LOGL, U = L / 8, S = SC::S;
  extern __shared__ float2 sm[];
  io.init(blockIdx.x, sm + LAY::ELEMS);
  const int tid = threadIdx.x;
  int t0, u0, t1, u1;
  if (MODE == MODE_ROW) {
    t0 = t1 = tid / U;
    u0 = u1 = tid % U;
  } else if (MODE == MODE_COL) {
    t0 = t1 = tid % T;
    u0 = u1 = tid / T;
  } else {
    t0 = tid / U;
    u0 = tid % U;
    t1 = tid % T;
    u1 = tid / T;
  }
  float2 v[8];
  int oidx[8];
  const bool valid0 = io.tile_valid(t0);
#pragma unroll
  for (int e = 0; e < 8; e++) v[e] = valid0 ? io.load(t0, u0 + e * U) : make_float2(0.f, 0.f);

  stage_compute<LOGL, SC::logr(0), 0, FWD>(v, u0, tw, oidx);
  if constexpr (S == 1) {
    if (valid0) io.store8(t0, u0, U, v);
    return;
  } else {
#pragma unroll
  for (int e = 0; e < 8; e++) sm[LAY::at(oidx[e], t0)] = v[e];
  __syncthreads();

  if constexpr (S >= 3) {
#pragma unroll
    for (int e = 0; e < 8; e++) v[e] = sm[LAY::at(u1 + e * U, t1)];
    __syncthreads();
    stage_compute<LOGL, SC::logr(1), SC::logns(1), FWD, MODE != MODE_ROW>(v, u1, tw, oidx);
#pragma unroll
    for (int e = 0; e < 8; e++) sm[LAY::at(oidx[e], t1)] = v[e];
    __syncthreads();
  }
  if constexpr (S >= 4) {
#pragma unroll
    for (int e = 0; e < 8; e++) v[e] = sm[LAY::at(u1 + e * U, t1)];
    __syncthreads();
    stage_compute<LOGL, SC::logr(2), SC::logns(2), FWD, MODE != MODE_ROW>(v, u1, tw, oidx);
#pragma unroll
    for (int e = 0; e < 8; e++) sm[LAY::at(oidx[e], t1)] = v[e];
    __syncthreads();
  }
  // last stage
#pragma unroll
  for (int e = 0; e < 8; e++) v[e] = sm[LAY::at(u1 + e * U, t1)];
  stage_compute<LOGL, SC::logr(S - 1), SC::logns(S - 1), FWD, MODE != MODE_ROW>(v, u1, tw, oidx);
  if (io.tile_valid(t1)) io.store8(t1, u1, U, v);
  }
}

// ---------------------------------------------------------------------------------
// IO functors
// ---------------------------------------------------------------------------------

// contiguous rows, in place or out of place; T rows per CTA
template <int LOGL, int T>
struct row_io {
  const float2* in;
  float2* out;
  size_t nrows;
  size_t row0;
  __device__ __forceinline__ void init(unsigned block, float2*) { row0 = (size_t)block * T; }
  __device__ __forceinline__ bool tile_valid(int t) const { return row0 + t < nrows; }
  __device__ __forceinline__ float2 load(int t, int pos) const {
    return in[((row0 + t) << LOGL) + pos];
  }
  __device__ __forceinline__ void store8(int t, int u, int U, float2 (&v)[8]) const {
    float2* o = out + ((row0 + t) << LOGL) + u;
#pragma unroll
    for (int e = 0; e < 8; e++) o[e * U] = v[e];
  }
};

// three-level twiddle table for W_n^idx, idx < n <= 2^30: idx = a*2^(2q) + b*2^q + c
struct big_twiddle {
  const float2* tab;  // [3][1 << q]: W^(c), W^(b << q), W^(a << 2q)
  int q;
};
__device__ __forceinline__ float2 big_tw_lookup(const float2* s, int q, uint32_t idx) {
  const uint32_t mask = (1u << q) - 1u;
  const float2 w0 = s[idx & mask];
  const float2 w1 = s[(1u << q) + ((idx >> q) & mask)];
  const float2 w2 = s[(2u << q) + (idx >> (2 * q))];
  return c_mul(c_mul(w2, w1), w0);
}

__device__ __forceinline__ float2 big_tw_lookup_ldg(const float2* __restrict__ g, int q, uint32_t idx) {
  const uint32_t mask = (1u << q) - 1u;
  const float2 w0 = __ldg(&g[idx & mask]);
  const float2 w1 = __ldg(&g[(1u << q) + ((idx >> q) & mask)]);
  const float2 w2 = __ldg(&g[(2u << q) + (idx >> (2 * q))]);
  return c_mul(c_mul(w2, w1), w0);
}

// column pass of a multi-pass transform: view [A][L][B], FFT along L for T adjacent b.
// store multiplies by the inter-pass twiddle W_{L*B}^{k*b} (forward table, conj if !FWD).
template <int LOGL, int T, bool FWD>
struct col_io {
  const float2* in;
  float2* out;
  size_t B;        // elements between consecutive FFT points
  uint32_t btiles; // B / T
  big_twiddle btw;
  size_t base;
  uint32_t b0;
  const float2* stw;
  __device__ __forceinline__ void init(unsigned block, float2* smem_extra) {
    const uint32_t a = block / btiles;
    b0 = (block % btiles) * T;
    base = ((size_t)a << LOGL) * B + b0;
    // stage the three small twiddle tables in shared memory
    float2* s = smem_extra;
    const int n = 3 << btw.q;
    for (int i = threadIdx.x; i < n; i += blockDim.x) s[i] = __ldg(&btw.tab[i]);
    stw = s;
    __syncthreads();
  }
  __device__ __forceinline__ bool tile_valid(int) const { return true; }
  __device__ __forceinline__ float2 load(int t, int pos) const { return in[base + (size_t)pos * B + t]; }
  __device__ __forceinline__ void store8(int t, int u, int U, float2 (&v)[8]) const {
    const uint32_t b = b0 + t;
    // twiddles W^{(u + e*U) * b}: base and ratio from the tables, powers by multiplication
    float2 wb = big_tw_lookup(stw, btw.q, (uint32_t)u * b);
    float2 r1 = big_tw_lookup(stw, btw.q, (uint32_t)U * b);
    if (!FWD) {
      wb.y = -wb.y;
      r1.y = -r1.y;
    }
    const float2 r2 = c_sqr(r1), r4 = c_sqr(r2);
    float2 w[8];
    w[0] = wb;
    w[1] = c_mul(wb, r1);
    w[2] = c_mul(wb, r2);
    w[3] = c_mul(w[1], r2);
    w[4] = c_mul(wb, r4);
    w[5] = c_mul(w[1], r4);
    w[6] = c_mul(w[2], r4);
    w[7] = c_mul(w[3], r4);
    float2* o = out + base + (size_t)u * B + t;
#pragma unroll
    for (int e = 0; e < 8; e++) o[(size_t)e * U * B] = c_mul(v[e], w[e]);
  }
};

// transposing last pass: rows [beta][k1][rest][L] -> natural order
//   in  row = beta*A + k1*S + rest            (A = n / L rows per transform, S = A / L1)
//   out idx = beta*n + k1 + L1*rest + A*k     (k = output index of this pass)
template <int LOGL, int T>
struct trans_io {
  const float2* in;
  float2* out;
  uint32_t A, S, L1;   // rows per transform, rest count, first-pass length
  uint32_t k1tiles;    // L1 / T
  size_t in_row0;      // row of t = 0
  size_t out0;         // out index of (t = 0, k = 0)
  __device__ __forceinline__ void init(unsigned block, float2*) {
    const uint32_t k1t = block % k1tiles;
    const uint32_t r = block / k1tiles;
    const uint32_t rest = r % S;
    const uint32_t beta = r / S;
    const uint32_t k1 = k1t * T;
    in_row0 = (size_t)beta * A + (size_t)k1 * S + rest;
    out0 = ((size_t)beta * A << LOGL) + k1 + (size_t)L1 * rest;
  }
  __device__ __forceinline__ bool tile_valid(int) const { return true; }
  __device__ __forceinline__ float2 load(int t, int pos) const {
    return in[((in_row0 + (size_t)t * S) << LOGL) + pos];
  }
  __device__ __forceinline__ void store8(int t, int u, int U, float2 (&v)[8]) const {
    float2* o = out + out0 + t + (size_t)A * u;
#pragma unroll
    for (int e = 0; e < 8; e++) o[(size_t)A * e * U] = v[e];
  }
};


// ---------------------------------------------------------------------------------
// TMA (cp.async.bulk) + mbarrier helpers
// ---------------------------------------------------------------------------------
// programmatic dependent launch (griddepcontrol): a kernel launched with the stream-serialisation attribute may start
// while its predecessor drains; everything it does before pdl_wait() (shared-memory tables, barrier set-up)
// overlaps the predecessor's tail, everything after sees the predecessor's results. No-ops in a normal launch.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// bounded wait: a TMA that never completes (bad tensor map) traps after ~2 s instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}
// 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ROW-mode transform as a persistent kernel: each CTA walks tiles of T contiguous rows; the next
// tile's rows are fetched by ONE cp.async.bulk (TMA) into the other shared-memory buffer while the
// current tile is transformed, so no thread ever waits on a global load in its critical path.
// Buffers: raw layout [T][L] as it arrives, then the padded exchange layout in place.
template <int LOGL, int T>
struct row_tma_smem {
  static constexpr int L = 1 << LOGL;
  static constexpr int BUF = T * (L + (L >> 4));  // elements per buffer (padded layout is the larger)
  // compact stage tables: stage s >= 1 needs W_{8^s * R}^k for k < 8^s  (8 + 64 + 512 entries at most)
  static constexpr int TW = (LOGL > 9) ? 584 : ((LOGL > 6) ? 72 : ((LOGL > 3) ? 8 : 0));
  static constexpr size_t bytes = 2 * (size_t)BUF * sizeof(float2) + 128 + (size_t)(TW + 8) * sizeof(float2);
};

// SK = true (process_block only) fuses the next two pipes into the epilogue while a whole row is in
// the CTA's registers: spectral kurtosis of the transformed row (K14/K15: zero it if flagged) and
// the detector's partial column sums of the surviving rows (K17 stage 1), one partial row per CTA.
struct row_sk_params {
  float thr_lo, thr_hi;   // scaled SK window (spectrum/rfi_mitigation.hpp:300-306)
  float* partial;         // [gridDim.x][ts_count]
  unsigned ts_count;      // time samples kept by the detector
};

template <int LOGL, int T, bool FWD, bool SK = false>
__global__ void __launch_bounds__(pass_threads<LOGL, T>::value,
                                  SK ? (pass_threads<LOGL, T>::min_blocks > 2 ? 2 : pass_threads<LOGL, T>::min_blocks)
                                     : pass_threads<LOGL, T>::min_blocks)
    fft_row_tma_kernel(const float2* __restrict__ in, float2* __restrict__ out, size_t nrows,
                       const float2* __restrict__ tw, row_sk_params skp) {
  using SC = sched<LOGL>;
  using LAY = tile_layout<LOGL, T, MODE_ROW>;
  constexpr int L = 1 << LOGL, U = L / 8, S = SC::S, BUF = row_tma_smem<LOGL, T>::BUF;
  extern __shared__ __align__(128) unsigned char smraw[];
  float2* const buf0 = reinterpret_cast<float2*>(smraw);
  float2* const buf1 = buf0 + BUF;
  uint64_t* const mbar = reinterpret_cast<uint64_t*>(buf1 + BUF);
  float2* const ctw = reinterpret_cast<float2*>(smraw + 2 * (size_t)BUF * sizeof(float2) + 128);
  const int tid = threadIdx.x;
  const int t = tid / U, u = tid % U;
  const unsigned ntiles = (unsigned)((nrows + T - 1) / T);
  if (tid == 0) {
    mbar_init(&mbar[0], 1);
    mbar_init(&mbar[1], 1);
    fence_mbar_init();
  }
  // compact stage twiddles: table of stage s (>= 1) starts at offset (8^s - 8) / 7 and holds
  // W_{Ns*R}^k = W_L^{k << (LOGL - 3s - logr(s))} for k < Ns = 8^s
  for (int s = 1; s < S; s++) {
    const int ns = 1 << (3 * s), off = (ns - 8) / 7, sh = LOGL - 3 * s - SC::logr(s);
    for (int k = tid; k < ns; k += blockDim.x) ctw[off + k] = __ldg(&tw[k << sh]);
  }
  __syncthreads();
  auto issue = [&](unsigned tl, int b) {  // one thread: fetch tile tl into buffer b
    const size_t row0 = (size_t)tl * T;
    const size_t rows = (nrows - row0 < (size_t)T) ? nrows - row0 : (size_t)T;
    const uint32_t bytes = (uint32_t)(rows << LOGL) * (uint32_t)sizeof(float2);
    fence_proxy_async();  // earlier generic-proxy accesses to this buffer are ordered before the async write
    mbar_expect_tx(&mbar[b], bytes);
    bulk_g2s(b ? buf1 : buf0, in + (row0 << LOGL), bytes, &mbar[b]);
  };
  float colacc[8];
#pragma unroll
  for (int e = 0; e < 8; e++) colacc[e] = 0.f;
  __shared__ float sk_s2[T][(U + 31) / 32], sk_s4[T][(U + 31) / 32];
  __shared__ int sk_zap[T];
  unsigned tile = blockIdx.x;
  if (tile < ntiles && tid == 0) issue(tile, 0);
  for (unsigned it = 0; tile < ntiles; tile += gridDim.x, it++) {
    const int b = it & 1;
    float2* const sm = b ? buf1 : buf0;
    const unsigned nxt = tile + gridDim.x;
    if (nxt < ntiles && tid == 0) issue(nxt, b ^ 1);
    mbar_wait(&mbar[b], (it >> 1) & 1);
    const size_t row = (size_t)tile * T + t;
    const bool valid = row < nrows;
    float2 v[8];
    int oidx[8];
#pragma unroll
    for (int e = 0; e < 8; e++) v[e] = valid ? sm[t * L + u + e * U] : make_float2(0.f, 0.f);
    stage_compute<LOGL, SC::logr(0), 0, FWD>(v, u, tw, oidx);
    if constexpr (S == 1) {
      if (valid) {
        float2* o = out + (row << LOGL) + u;
#pragma unroll
        for (int e = 0; e < 8; e++) o[e * U] = v[e];
      }
      __syncthreads();  // buffer b may be refilled from the next iteration on
    } else {
      __syncthreads();  // every raw read done before the padded layout overwrites the buffer
#pragma unroll
      for (int e = 0; e < 8; e++) sm[LAY::at(oidx[e], t)] = v[e];
      __syncthreads();
      if constexpr (S >= 3) {
#pragma unroll
        for (int e = 0; e < 8; e++) v[e] = sm[LAY::at(u + e * U, t)];
        __syncthreads();
        stage_compute<LOGL, SC::logr(1), SC::logns(1), FWD, false, 0, false>(v, u, ctw + 0, oidx);
#pragma unroll
        for (int e = 0; e < 8; e++) sm[LAY::at(oidx[e], t)] = v[e];
        __syncthreads();
      }
      if constexpr (S >= 4) {
#pragma unroll
        for (int e = 0; e < 8; e++) v[e] = sm[LAY::at(u + e * U, t)];
        __syncthreads();
        stage_compute<LOGL, SC::logr(2), SC::logns(2), FWD, false, 0, false>(v, u, ctw + 8, oidx);
#pragma unroll
        for (int e = 0; e < 8; e++) sm[LAY::at(oidx[e], t)] = v[e];
        __syncthreads();
      }
#pragma unroll
      for (int e = 0; e < 8; e++) v[e] = sm[LAY::at(u + e * U, t)];
      stage_compute<LOGL, SC::logr(S - 1), SC::logns(S - 1), FWD, false, 0, false>(v, u, ctw + ((1 << (3 * (S - 1))) - 8) / 7, oidx);
      if constexpr (SK) {
        static_assert(!SK || U >= 32, "SK fusion needs at least one warp per row");
        float pw[8], s2 = 0.f, s4 = 0.f;
#pragma unroll
        for (int e = 0; e < 8; e++) {
          pw[e] = valid ? (v[e].x * v[e].x + v[e].y * v[e].y) : 0.f;
          s2 += pw[e];
          s4 += pw[e] * pw[e];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          s2 += __shfl_xor_sync(0xffffffffu, s2, o);
          s4 += __shfl_xor_sync(0xffffffffu, s4, o);
        }
        if ((tid & 31) == 0) {
          sk_s2[t][u >> 5] = s2;
          sk_s4[t][u >> 5] = s4;
        }
        __syncthreads();
        if (u == 0) {
          float a = 0.f, bsum = 0.f;
          for (int w = 0; w < (U + 31) / 32; w++) {  // fixed order
            a += sk_s2[t][w];
            bsum += sk_s4[t][w];
          }
          const float sk = (float)L * (bsum / (a * a));
          sk_zap[t] = (sk > skp.thr_hi || sk < skp.thr_lo) ? 1 : 0;  // NaN (all-zero row): untouched
        }
        __syncthreads();
        const bool zap = sk_zap[t] != 0;
        if (valid) {
          float2* o = out + (row << LOGL) + u;
#pragma unroll
          for (int e = 0; e < 8; e++) o[e * U] = zap ? make_float2(0.f, 0.f) : v[e];
          if (!zap) {
#pragma unroll
            for (int e = 0; e < 8; e++) colacc[e] += pw[e];
          }
        }
      } else {
        if (valid) {
          float2* o = out + (row << LOGL) + u;
#pragma unroll
          for (int e = 0; e < 8; e++) o[e * U] = v[e];
        }
      }
      __syncthreads();  // all reads of buffer b done: it may be refilled from the next iteration on
    }
  }
  if constexpr (SK) {
    float* const red = reinterpret_cast<float*>(buf0);  // tile buffers are free now
    __syncthreads();
#pragma unroll
    for (int e = 0; e < 8; e++) red[t * L + u + e * U] = colacc[e];
    __syncthreads();
    for (int c = tid; c < L; c += blockDim.x) {
      float a = 0.f;
      for (int tt = 0; tt < T; tt++) a += red[tt * L + c];
      if ((unsigned)c < skp.ts_count) skp.partial[(size_t)blockIdx.x * skp.ts_count + c] = a;
    }
  }
}


// K12 chirp factor (S/coherent_dedispersion.hpp:133-150 phase_factor_v3): f = f_min + df*i in fp64,
// k = (D*1e6*dm)/f * ((f-f_c)/f_c)^2, factor = exp(-2 pi i frac(k)); used by dedisperse_kernel and by the
// waterfall kernel that fuses s1 + chirp into its load (CHIRP = true below).
__device__ __forceinline__ float2 chirp_factor(double f_min, double df, double inv_fc, double f_c,
                                               double ddm, unsigned i) {
  // 1/f by __drcp_rn (correctly rounded) and (f - f_c) * (1/f_c): each differs from the reference's
  // true divisions by <= 1 ulp of fp64, i.e. <= |k| * 2.2e-16 cycles of phase (DESIGN.md section 4)
  const double f = fma(df, (double)i, f_min);
  const double q = (f - f_c) * inv_fc;
  const double k = (ddm * __drcp_rn(f)) * (q * q);
  const float frac = (float)(k - trunc(k));
  float s, c;
  sincospif(-2.0f * frac, &s, &c);
  return make_float2(c, s);
}

struct row_chirp_params {
  double f_min, df, inv_fc, f_c, ddm;
  const float* mean;      // mean |X|^2 of the block (s1 statistic), finalised by the preceding kernel
  float threshold, coef;  // s1: zap above threshold * mean, scale the rest by coef
  int newton;             // whole-row kernel: reciprocal mode = the kernel's CHIRP template value (1, 3, 4; 2 = exact)
  // optional: -2 pi frac(k) of every bin of the block (chirp_phase_table_kernel); the whole-row kernel then runs as
  // CHIRP = 5 and evaluates no fp64 at all
  const float* phase;
};

#ifndef SRTB_FAST_SINCOS
#define SRTB_FAST_SINCOS 1
#endif

// s1 + chirp on one spectrum bin: f and 1/f in fp64 (K12: coherent_dedispersion.hpp:133-150)
__device__ __forceinline__ float2 chirp_point(float2 v, double f, double r, const row_chirp_params& cp,
                                                     float limit) {
  const double q = (f - cp.f_c) * cp.inv_fc;
  const double k = (cp.ddm * r) * (q * q);
  // k mod 1 in [-0.5, 0.5]: e^{-2 pi i k} is unchanged by the integer that is dropped
  constexpr double MAGIC = 6755399441055744.0;  // 1.5 * 2^52
  const double kr = __dadd_rn(__dadd_rn(k, MAGIC), -MAGIC);
  const float frac = (float)(k - kr);
  float s, c;
#if SRTB_FAST_SINCOS
  __sincosf(-6.283185307179586f * frac, &s, &c);  // SFU, argument in [-pi, pi]: abs error <= 2^-21
#else
  sincospif(-2.0f * frac, &s, &c);
#endif
  const float scale = (v.x * v.x + v.y * v.y > limit) ? 0.f : cp.coef;  // rfi_mitigation_pipe.hpp:66-79
  const float wr = c * scale, wi = s * scale;
  return make_float2(v.x * wr - v.y * wi, v.x * wi + v.y * wr);
}

// the same on a tabulated phase: ang = -2 pi frac(k) in [-pi, pi], rounded to fp32 once
__device__ __forceinline__ float2 chirp_point_tab(float2 v, float ang, float limit, float coef) {
  float s, c;
  __sincosf(ang, &s, &c);
  const float scale = (v.x * v.x + v.y * v.y > limit) ? 0.f : coef;
  const float wr = c * scale, wi = s * scale;
  return make_float2(v.x * wr - v.y * wi, v.x * wi + v.y * wr);
}

// K12 phase of bin `bin` (an integer, exact in fp64): k exactly as chirp_factor evaluates it (fp64, correctly rounded
// reciprocal), reduced to [-1/2, 1/2] cycles, as the fp32 angle -2 pi frac(k) — the very value chirp_point hands to
// the SFU, so every route that takes its angle from here agrees with it to the last bit of the argument
__device__ __forceinline__ float chirp_angle(double bin, double f_min, double df, double inv_fc, double f_c, double ddm) {
  const double f = fma(df, bin, f_min);
  const double q = (f - f_c) * inv_fc;
  const double k = (ddm * __drcp_rn(f)) * (q * q);
  const float fr = (float)(k - rint(k));  // the difference is exact, in [-1/2, 1/2]
  return -6.283185307179586f * fr;
}

// chirp_angle of every bin of a block, once per (block geometry, DM). DM and band are constants of a run, so the table
// is part of the plan like the twiddles.
__global__ void __launch_bounds__(256) chirp_phase_table_kernel(float* __restrict__ out, size_t n, double f_min,
                                                                double df, double inv_fc, double f_c, double ddm) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = chirp_angle((double)i, f_min, df, inv_fc, f_c, ddm);
}

// ---------------------------------------------------------------------------------
// Row pass with sixteen points per thread (radix-16 stages: L = 4096 as 16^3, 2048 as 16*16*8,
// 1024 as 16*16*4, 256 as 16*16): three stages and five CTA barriers per 4096-point row instead of
// four and eight. Lanes run along the FFT index, so a thread reads W^k, W^2k, W^4k of its butterfly from
// compact per-stage tables and forms the other powers by at most two further multiplications.
// The exchange layout is an XOR swizzle (idx ^ ((idx >> 4) & 15)): conflict-free for every stage's
// reads and writes without padding, so the tile buffers stay at exactly T*L elements.
// ---------------------------------------------------------------------------------
template <int LOGL>
struct row16_t {
  static constexpr int value = (LOGL >= 12) ? 1 : (1 << (12 - LOGL));  // 4096 points, 256 threads per tile
};
template <int LOGL, int T>
struct row16_smem {
  static constexpr int L = 1 << LOGL;
  static constexpr int BUF = T * L;
  static constexpr int S = sched16<LOGL>::S;
  // stage s >= 1: three tables (W^k, W^2k, W^4k) of Ns = 2^logns(s) entries
  static constexpr int TW = 3 * ((1 << sched16<LOGL>::logns(1)) + (S > 2 ? (1 << sched16<LOGL>::logns(2)) : 0));
  static constexpr size_t bytes = 2 * (size_t)BUF * sizeof(float2) + 128 + (size_t)(TW + 8) * sizeof(float2);
};

__device__ __forceinline__ int row16_sw(int idx) { return idx ^ ((idx >> 4) & 15); }

template <int LOGL, int LOGR, int LOGNS, bool FWD>
__device__ __forceinline__ void stage_compute16_row(float2 (&v)[16], int u, const float2* __restrict__ ctw,
                                                    int (&oidx)[16]) {
  constexpr int L = 1 << LOGL, U = L / 16, R = 1 << LOGR, NB = 16 / R, NS = 1 << LOGNS;
  static_assert(LOGR >= 2 && LOGR <= 4, "radix 4, 8 or 16");
#pragma unroll
  for (int m = 0; m < NB; m++) {
    const int b = u + m * U;
    const int k = b & (NS - 1);
    if constexpr (LOGNS > 0) {
      const float2 w1 = c_dir<FWD>(ctw[k]), w2 = c_dir<FWD>(ctw[NS + k]);
      const float2 w3 = c_mul(w1, w2);
      v[m + NB] = c_mul(v[m + NB], w1);
      v[m + 2 * NB] = c_mul(v[m + 2 * NB], w2);
      v[m + 3 * NB] = c_mul(v[m + 3 * NB], w3);
      if constexpr (R >= 8) {
        const float2 w4 = c_dir<FWD>(ctw[2 * NS + k]);
        const float2 w5 = c_mul(w4, w1), w6 = c_mul(w4, w2), w7 = c_mul(w4, w3);
        v[m + 4 * NB] = c_mul(v[m + 4 * NB], w4);
        v[m + 5 * NB] = c_mul(v[m + 5 * NB], w5);
        v[m + 6 * NB] = c_mul(v[m + 6 * NB], w6);
        v[m + 7 * NB] = c_mul(v[m + 7 * NB], w7);
        if constexpr (R == 16) {
          const float2 w8 = c_sqr(w4);
          v[8] = c_mul(v[8], w8);
          v[9] = c_mul(v[9], c_mul(w8, w1));
          v[10] = c_mul(v[10], c_mul(w8, w2));
          v[11] = c_mul(v[11], c_mul(w8, w3));
          v[12] = c_mul(v[12], c_mul(w8, w4));
          v[13] = c_mul(v[13], c_mul(w8, w5));
          v[14] = c_mul(v[14], c_mul(w8, w6));
          v[15] = c_mul(v[15], c_mul(w8, w7));
        }
      }
    }
    if constexpr (R == 16) {
      dft16<FWD>(v);
    } else if constexpr (R == 8) {
      dft8<FWD>(v[m], v[m + 2], v[m + 4], v[m + 6], v[m + 8], v[m + 10], v[m + 12], v[m + 14]);
    } else {
      dft4<FWD>(v[m], v[m + 4], v[m + 8], v[m + 12]);
    }
    const int obase = ((b >> LOGNS) << (LOGNS + LOGR)) + k;
#pragma unroll
    for (int i = 0; i < R; i++) oidx[m + i * NB] = obase + i * NS;
  }
}

template <int LOGL, int T, bool FWD, bool SK = false, bool CHIRP = false>
__global__ void __launch_bounds__(((1 << LOGL) / 16) * T, 3)
    fft_row16_tma_kernel(const float2* __restrict__ in, float2* __restrict__ out, size_t nrows,
                         const float2* __restrict__ tw, row_sk_params skp, row_chirp_params cp) {
  using SC = sched16<LOGL>;
  constexpr int L = 1 << LOGL, U = L / 16, S = SC::S, BUF = row16_smem<LOGL, T>::BUF;
  static_assert(S == 2 || S == 3, "64 <= L <= 4096");
  extern __shared__ __align__(128) unsigned char smraw[];
  float2* const buf0 = reinterpret_cast<float2*>(smraw);
  float2* const buf1 = buf0 + BUF;
  uint64_t* const mbar = reinterpret_cast<uint64_t*>(buf1 + BUF);
  float2* const ctw = reinterpret_cast<float2*>(smraw + 2 * (size_t)BUF * sizeof(float2) + 128);
  const int tid = threadIdx.x;
  const int t = tid / U, u = tid % U;
  const unsigned ntiles = (unsigned)((nrows + T - 1) / T);
  if (tid == 0) {
    mbar_init(&mbar[0], 1);
    mbar_init(&mbar[1], 1);
    fence_mbar_init();
  }
  // stage s >= 1 (Ns = 16^s, radix R): tables p = 1, 2, 4 of W_{Ns*R}^{k p} = W_L^{(k p) << (LOGL - 4s - logr)}
  constexpr int OFF2 = 3 << SC::logns(1);  // table offset of the third stage
#pragma unroll
  for (int s = 1; s < S; s++) {
    const int ns = 1 << SC::logns(s), off = (s == 1) ? 0 : OFF2, sh = LOGL - SC::logns(s) - SC::logr(s);
    for (int i = tid; i < 3 * ns; i += blockDim.x) {
      const int p = i / ns, k = i - p * ns;
      ctw[off + i] = __ldg(&tw[(k << p) << sh]);
    }
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();  // the spectrum and the s1 mean come from the preceding kernels
  auto issue = [&](unsigned tl, int b) {
    const size_t row0 = (size_t)tl * T;
    const size_t rows = (nrows - row0 < (size_t)T) ? nrows - row0 : (size_t)T;
    const uint32_t bytes = (uint32_t)(rows << LOGL) * (uint32_t)sizeof(float2);
    fence_proxy_async();
    mbar_expect_tx(&mbar[b], bytes);
    bulk_g2s(b ? buf1 : buf0, in + (row0 << LOGL), bytes, &mbar[b]);
  };
  float colacc[SK ? 16 : 1];
#pragma unroll
  for (int e = 0; e < (SK ? 16 : 1); e++) colacc[e] = 0.f;
  __shared__ float sk_s2[2][T][(U + 31) / 32], sk_s4[2][T][(U + 31) / 32];
  unsigned tile = blockIdx.x;
  if (tile < ntiles && tid == 0) issue(tile, 0);
  for (unsigned it = 0; tile < ntiles; tile += gridDim.x, it++) {
    const int b = it & 1;
    float2* const sm = (b ? buf1 : buf0) + t * L;
    const unsigned nxt = tile + gridDim.x;
    if (nxt < ntiles && tid == 0) issue(nxt, b ^ 1);
    mbar_wait(&mbar[b], (it >> 1) & 1);
    const size_t row = (size_t)tile * T + t;
    const bool valid = row < nrows;
    float2 v[16];
    int oidx[16];
#pragma unroll
    for (int e = 0; e < 16; e++) v[e] = valid ? sm[u + e * U] : make_float2(0.f, 0.f);
    if constexpr (CHIRP) {
      // rfi_mitigation_s1 (zap + normalise, rfi_mitigation_pipe.hpp:66-79) and the dedispersion chirp
      // (coherent_dedispersion.hpp:223-237) applied to the spectrum on its way into the waterfall FFT
      const float limit = cp.threshold * __ldg(cp.mean);
      if (cp.phase != nullptr) {
        // tabulated phases (block path): consecutive lanes read consecutive entries
        const float* const ph = cp.phase + (valid ? (row << LOGL) + u : 0);
        float ang[16];
#pragma unroll
        for (int e = 0; e < 16; e++) ang[e] = __ldg(ph + e * U);
#pragma unroll
        for (int e = 0; e < 16; e++) v[e] = chirp_point_tab(v[e], ang[e], limit, cp.coef);
      } else {
#pragma unroll
        for (int e = 0; e < 16; e++) {
          float2 a = v[e];
          if (a.x * a.x + a.y * a.y > limit) a = make_float2(0.f, 0.f);
          else a = make_float2(a.x * cp.coef, a.y * cp.coef);
          const float2 w = chirp_factor(cp.f_min, cp.df, cp.inv_fc, cp.f_c, cp.ddm, (unsigned)((row << LOGL) + u + e * U));
          v[e] = make_float2(a.x * w.x - a.y * w.y, a.x * w.y + a.y * w.x);
        }
      }
    }
    stage_compute16_row<LOGL, SC::logr(0), 0, FWD>(v, u, ctw, oidx);
    __syncthreads();  // every linear read done before the swizzled layout overwrites the buffer
#pragma unroll
    for (int e = 0; e < 16; e++) sm[row16_sw(oidx[e])] = v[e];
    __syncthreads();
    if constexpr (S == 3) {
#pragma unroll
      for (int e = 0; e < 16; e++) v[e] = sm[row16_sw(u + e * U)];
      __syncthreads();
      stage_compute16_row<LOGL, SC::logr(1), SC::logns(1), FWD>(v, u, ctw, oidx);
#pragma unroll
      for (int e = 0; e < 16; e++) sm[row16_sw(oidx[e])] = v[e];
      __syncthreads();
    }
#pragma unroll
    for (int e = 0; e < 16; e++) v[e] = sm[row16_sw(u + e * U)];
    stage_compute16_row<LOGL, SC::logr(S - 1), SC::logns(S - 1), FWD>(v, u, ctw + ((S == 3) ? OFF2 : 0), oidx);
    if constexpr (SK) {
      static_assert(!SK || U >= 32, "SK fusion needs at least one warp per row");
      float s2 = 0.f, s4 = 0.f;
#pragma unroll
      for (int e = 0; e < 16; e++) {
        const float pw = valid ? (v[e].x * v[e].x + v[e].y * v[e].y) : 0.f;
        s2 += pw;
        s4 += pw * pw;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
        s4 += __shfl_xor_sync(0xffffffffu, s4, o);
      }
      // per-warp partials alternate between two slots so that one barrier per tile is enough
      float(*const ps2)[(U + 31) / 32] = sk_s2[it & 1];
      float(*const ps4)[(U + 31) / 32] = sk_s4[it & 1];
      if ((tid & 31) == 0) {
        ps2[t][u >> 5] = s2;
        ps4[t][u >> 5] = s4;
      }
      __syncthreads();
      bool zap;
      {
        // every warp folds the row's NW per-warp partials with the same fixed shuffle tree
        constexpr int NW = (U + 31) / 32;
        const int lane = tid & 31;
        float a = (lane < NW) ? ps2[t][lane] : 0.f, bsum = (lane < NW) ? ps4[t][lane] : 0.f;
#pragma unroll
        for (int o = NW / 2; o > 0; o >>= 1) {
          a += __shfl_xor_sync(0xffffffffu, a, o);
          bsum += __shfl_xor_sync(0xffffffffu, bsum, o);
        }
        a = __shfl_sync(0xffffffffu, a, 0);
        bsum = __shfl_sync(0xffffffffu, bsum, 0);
        const float sk = (float)L * (bsum / (a * a));
        zap = (sk > skp.thr_hi || sk < skp.thr_lo);  // NaN (all-zero row): untouched
      }
      if (valid) {
        float2* o = out + (row << LOGL) + u;
#pragma unroll
        for (int e = 0; e < 16; e++) o[e * U] = zap ? make_float2(0.f, 0.f) : v[e];
        if (!zap) {
#pragma unroll
          for (int e = 0; e < 16; e++) colacc[e] += v[e].x * v[e].x + v[e].y * v[e].y;
        }
      }
    } else {
      if (valid) {
        float2* o = out + (row << LOGL) + u;
#pragma unroll
        for (int e = 0; e < 16; e++) o[e * U] = v[e];
      }
    }
    __syncthreads();  // all reads of buffer b done: it may be refilled from the next iteration on
  }
  if constexpr (SK) {
    float* const red = reinterpret_cast<float*>(buf0);  // tile buffers are free now
    __syncthreads();
#pragma unroll
    for (int e = 0; e < 16; e++) red[t * L + u + e * U] = colacc[e];
    __syncthreads();
    for (int c = tid; c < L; c += blockDim.x) {
      float a = 0.f;
      for (int tt = 0; tt < T; tt++) a += red[tt * L + c];
      if ((unsigned)c < skp.ts_count) skp.partial[(size_t)blockIdx.x * skp.ts_count + c] = a;
    }
  }
}


// ---------------------------------------------------------------------------------
// COL and TRANS passes fed by tensor-map TMA (cp.async.bulk.tensor, SASS: UTMALDG)
// ---------------------------------------------------------------------------------
struct alignas(64) tensor_map_blob {
  unsigned char bytes[128];  // a CUtensorMap, passed by value as a __grid_constant__ parameter
};

__device__ __forceinline__ void tma_load_2d(void* dst_smem, const tensor_map_blob* tmap, int c0, int c1,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          smem_u32(dst_smem)),
      "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst_smem, const tensor_map_blob* tmap, int c0, int c1, int c2,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
          smem_u32(dst_smem)),
      "l"(tmap), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
      : "memory");
}

template <int LOGL, int T>
struct tile_tma_smem {
  static constexpr int L = 1 << LOGL;
  static constexpr int BUF = T * L;  // elements per buffer (COL / TRANS layouts are dense)
  static constexpr size_t data_bytes = 2 * (size_t)BUF * sizeof(float2);
  // [2 tile buffers][128 B: mbarriers][stage twiddles W_L^j, L entries][3 << q inter-pass twiddles]
  static constexpr size_t bytes(int q) { return data_bytes + 128 + (size_t)(L + (3 << q)) * sizeof(float2); }
};

// raw-fused sixteen-point first sweep: [exchange tile][2 raw byte tiles of L x 4T bytes][128 B: mbarriers][stage
// twiddles]; the inter-sweep tables stay in global memory (two look-ups per thread and tile, fetched before the
// stages run) so that three CTAs fit an SM at L = 512. With T = 8 a row of the exchange tile is 64 bytes — half the
// banks — and the four rows a warp writes after a radix-16 stage would all have the same parity: one spare row
// after every sixteen (tile rows r -> r + (r >> 4)) spreads them again.
// From L = 2048 (a 128 KiB exchange tile) ONE raw tile buffer is kept: stage 0 decodes the tile into registers at the
// start, so the next tile lands in the same buffer while the stages run (one CTA per SM at 1024 threads).
template <int LOGL, int T>
struct raw16_smem {
  static constexpr int L = 1 << LOGL;
  static constexpr int BUF = T * L;
  static constexpr bool PAD = (T == 8) && ((L / 16) % 16 == 0);
  static constexpr int XBUF = PAD ? BUF + BUF / 16 : BUF;
  static constexpr int NRAW = (LOGL >= 11) ? 1 : 2;
  static constexpr size_t bytes = (size_t)XBUF * sizeof(float2) + NRAW * (size_t)BUF * 4 + 128 + (size_t)L * sizeof(float2);
};

// the same two measures for the plain (complex input) sixteen-point column sweep with 64-byte tile rows: both TMA
// buffers get the spare rows (the tile lands dense, the exchange uses the padded rows), the inter-sweep tables stay in
// global memory, three CTAs per SM at L = 512. Not for the chirp-on-load variant (two CTAs per SM by registers).
template <int LOGL, int T, bool CH>
struct col16_smem {
  static constexpr int L = 1 << LOGL;
  static constexpr int BUF = T * L;
  static constexpr bool PAD = raw16_smem<LOGL, T>::PAD && !CH;
  static constexpr size_t bytes(int q) {
    return PAD ? 2 * (size_t)(BUF + BUF / 16) * sizeof(float2) + 128 + (size_t)L * sizeof(float2)
               : tile_tma_smem<LOGL, T>::bytes(q);
  }
};

// Column pass, persistent: view [A][L][B] (B = elements between consecutive FFT points). A tile is the
// L x T box at (row a*L, column b0) of the 2-D tensor [A*L][B]; ONE TMA box load (per 256 rows) brings
// it into shared memory in exactly the column-mode layout [idx][t], double buffered across tiles.
// Stores go straight from registers with the inter-pass twiddle W_{L*B}^{k b} applied.
// The raw first pass (unpack fused in) exists on the sixteen-point kernel only (fft_col16_tma_kernel, RAW != 0):
// the tensor map then describes the 8-bit baseband bytes, a tile is L x (T*G) bytes
// (G = bytes per complex point: 2 for one stream, 4 when two streams share the block) and stage 0
// converts the two samples at byte offsets o0/o1 of each group to float (K1's integer -> f32 cast,
// exact) instead of reading complex64 that a separate kernel would have written and this one re-read.
// RAW == 3: packed sub-byte samples (2 or 4 bits, MSB first, unsigned: unpack.hpp:43-156): a complex point is 2*bits
// consecutive bits. `delta`: byte offset subtracted for odd points (gznupsr_a1 puts four consecutive samples of one
// stream into a word, so odd points sit 2 bytes after the even point of the same word, not G bytes: unpack.hpp:338-369)
struct raw_params {
  int G, o0, o1;
  int delta;      // RAW 1/2: offset correction of odd points
  int row_bytes;  // bytes of one tile row in shared memory (T * G, or T * bits / 4 for packed samples)
  int bits;       // RAW 3: bits per sample
};

template <int LOGL, int T, bool FWD>
__global__ void __launch_bounds__(pass_threads<LOGL, T>::value, pass_threads<LOGL, T>::min_blocks)
    fft_col_tma_kernel(const __grid_constant__ tensor_map_blob tmap, float2* __restrict__ out, size_t B,
                       uint32_t btiles, uint32_t ntiles, big_twiddle btw, const float2* __restrict__ tw) {
  using SC = sched<LOGL>;
  constexpr int L = 1 << LOGL, U = L / 8, S = SC::S, BUF = tile_tma_smem<LOGL, T>::BUF;
  constexpr int ROWS_PER_BOX = (L < 256) ? L : 256;
  extern __shared__ __align__(128) unsigned char smraw[];
  float2* const buf0 = reinterpret_cast<float2*>(smraw);
  float2* const buf1 = buf0 + BUF;
  uint64_t* const mbar = reinterpret_cast<uint64_t*>(buf1 + BUF);
  float2* const ltw = reinterpret_cast<float2*>(smraw + tile_tma_smem<LOGL, T>::data_bytes + 128);
  float2* const stw = ltw + L;
  const int tid = threadIdx.x;
  const int t = tid % T, u = tid / T;
  if (tid == 0) {
    mbar_init(&mbar[0], 1);
    mbar_init(&mbar[1], 1);
    fence_mbar_init();
  }
  for (int i = tid; i < (3 << btw.q); i += blockDim.x) stw[i] = __ldg(&btw.tab[i]);
  for (int i = tid; i < L; i += blockDim.x) ltw[i] = __ldg(&tw[i]);
  __syncthreads();
  auto issue = [&](uint32_t tl, int b) {
    const uint32_t a = tl / btiles, b0 = (tl % btiles) * T;
    fence_proxy_async();
    float2* dst = b ? buf1 : buf0;
    mbar_expect_tx(&mbar[b], (uint32_t)(BUF * sizeof(float2)));
#pragma unroll
    for (int r = 0; r < L; r += ROWS_PER_BOX)
      tma_load_2d(dst + r * T, &tmap, (int)b0, (int)(a * L + r), &mbar[b]);
  };
  uint32_t tile = blockIdx.x;
  if (tile < ntiles && tid == 0) issue(tile, 0);
  for (uint32_t it = 0; tile < ntiles; tile += gridDim.x, it++) {
    const int b = it & 1;
    float2* const sm = b ? buf1 : buf0;
    const uint32_t nxt = tile + gridDim.x;
    if (nxt < ntiles && tid == 0) issue(nxt, b ^ 1);
    mbar_wait(&mbar[b], (it >> 1) & 1);
    float2 v[8];
    int oidx[8];
#pragma unroll
    for (int e = 0; e < 8; e++) v[e] = sm[(u + e * U) * T + t];
    stage_compute<LOGL, SC::logr(0), 0, FWD>(v, u, tw, oidx);
    if constexpr (S > 1) {
      __syncthreads();
#pragma unroll
      for (int e = 0; e < 8; e++) sm[oidx[e] * T + t] = v[e];
      __syncthreads();
      if constexpr (S >= 3) {
#pragma unroll
        for (int e = 0; e < 8; e++) v[e] = sm[(u + e * U) * T + t];
        __syncthreads();
        stage_compute<LOGL, SC::logr(1), SC::logns(1), FWD, true, LOGL - SC::logns(1) - SC::logr(1), false>(v, u, ltw, oidx);
#pragma unroll
        for (int e = 0; e < 8; e++) sm[oidx[e] * T + t] = v[e];
        __syncthreads();
      }
      if constexpr (S >= 4) {
#pragma unroll
        for (int e = 0; e < 8; e++) v[e] = sm[(u + e * U) * T + t];
        __syncthreads();
        stage_compute<LOGL, SC::logr(2), SC::logns(2), FWD, true, LOGL - SC::logns(2) - SC::logr(2), false>(v, u, ltw, oidx);
#pragma unroll
        for (int e = 0; e < 8; e++) sm[oidx[e] * T + t] = v[e];
        __syncthreads();
      }
#pragma unroll
      for (int e = 0; e < 8; e++) v[e] = sm[(u + e * U) * T + t];
      stage_compute<LOGL, SC::logr(S - 1), SC::logns(S - 1), FWD, true, LOGL - SC::logns(S - 1) - SC::logr(S - 1), false>(v, u, ltw, oidx);
    }
    {
      // store k = u + e*U of column b0 + t, times W_{L*B}^{k (b0 + t)}
      const uint32_t a = tile / btiles, b0 = (tile % btiles) * T;
      const uint32_t bb = b0 + t;
      float2 wb = big_tw_lookup(stw, btw.q, (uint32_t)u * bb);
      float2 r1 = big_tw_lookup(stw, btw.q, (uint32_t)U * bb);
      if (!FWD) {
        wb.y = -wb.y;
        r1.y = -r1.y;
      }
      const float2 r2 = c_sqr(r1), r4 = c_sqr(r2);
      float2 w[8];
      w[0] = wb;
      w[1] = c_mul(wb, r1);
      w[2] = c_mul(wb, r2);
      w[3] = c_mul(w[1], r2);
      w[4] = c_mul(wb, r4);
      w[5] = c_mul(w[1], r4);
      w[6] = c_mul(w[2], r4);
      w[7] = c_mul(w[3], r4);
      float2* o = out + ((size_t)a << LOGL) * B + b0 + (size_t)u * B + t;
#pragma unroll
      for (int e = 0; e < 8; e++) o[(size_t)e * U * B] = c_mul(v[e], w[e]);
    }
    __syncthreads();  // buffer b may be refilled from the next iteration on
  }
}

// Column pass with sixteen points per thread and radix-16 stages (two stages: L = 256 as 16 x 16, L = 128 as
// 16 x 8): one shared-memory exchange and three CTA barriers per tile instead of two and five. Same tiles,
// tensor maps, twiddle tables and results (up to fp32 rounding) as fft_col_tma_kernel.
template <int LOGL, int T>
struct col16_threads {
  static constexpr int value = ((1 << LOGL) / 16) * T;
  static constexpr int min_blocks = (768 / value) < 1 ? 1 : (768 / value);  // aim at 24 resident warps per SM
};

// CH (long waterfall rows, process_block only): rfi_mitigation_s1 (zap + normalise) and the dedispersion chirp are
// applied to the spectrum as the tile's points are taken out of shared memory (the bin of point idx of column b0 + t
// of row a is a L B + idx B + b0 + t); 1/f by Newton steps from the point U B bins below (cp.newton = 1 or 2 steps,
// else the exact reciprocal), like the whole-row kernel.
template <int LOGL, int T, bool FWD, int RAW, bool CH>
__device__ __forceinline__ void col16_body(const tensor_map_blob* tmap_, float2* __restrict__ out, size_t B,
                                           uint32_t btiles, uint32_t ntiles, const big_twiddle& btw,
                                           const float2* __restrict__ tw, const raw_params& rp,
                                           const row_chirp_params& cp) {
  const tensor_map_blob& tmap = *tmap_;
  using SC = sched16<LOGL>;
  constexpr int L = 1 << LOGL, U = L / 16, S = SC::S, BUF = tile_tma_smem<LOGL, T>::BUF;
  constexpr int ROWS_PER_BOX = (L < 256) ? L : 256;
  // exchange tile with a spare row per sixteen (raw16_smem / col16_smem); with it the inter-sweep tables stay global
  constexpr bool PADX = (RAW != 0) ? raw16_smem<LOGL, T>::PAD : col16_smem<LOGL, T, CH>::PAD;
  constexpr bool STWG = (RAW != 0) || PADX;
  constexpr int XBUF = PADX ? BUF + BUF / 16 : BUF;
  constexpr int UP = PADX ? U + U / 16 : U;                         // distance of a thread's sixteen slots
  extern __shared__ __align__(128) unsigned char smraw[];
  float2* const buf0 = reinterpret_cast<float2*>(smraw);
  float2* const buf1 = buf0 + XBUF;
  constexpr bool ONE_RAW = (RAW != 0) && raw16_smem<LOGL, T>::NRAW == 1;
  unsigned char* const raw0 = reinterpret_cast<unsigned char*>(buf1);
  unsigned char* const raw1 = ONE_RAW ? raw0 : raw0 + (size_t)BUF * 4;
  // RAW: right after the raw tiles (4 BUF bytes = BUF / 2 elements each); else after the second tile buffer
  uint64_t* const mbar = reinterpret_cast<uint64_t*>(buf1 + ((RAW != 0) ? raw16_smem<LOGL, T>::NRAW * BUF / 2 : XBUF));
  float2* const ltw = reinterpret_cast<float2*>(reinterpret_cast<unsigned char*>(mbar) + 128);
  const float2* const stw = STWG ? btw.tab : ltw + L;
  const int tid = threadIdx.x;
  const int t = tid % T, u = tid / T;
  if (tid == 0) {
    mbar_init(&mbar[0], 1);
    mbar_init(&mbar[1], 1);
    fence_mbar_init();
  }
  if constexpr (!STWG)
    for (int i = tid; i < (3 << btw.q); i += blockDim.x) ltw[L + i] = __ldg(&btw.tab[i]);
  for (int i = tid; i < L; i += blockDim.x) ltw[i] = __ldg(&tw[i]);
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();  // the input (and, in place, the output region) belongs to the preceding kernel until here
  auto issue = [&](uint32_t tl, int b) {
    const uint32_t a = tl / btiles, b0 = (tl % btiles) * T;
    fence_proxy_async();
    if constexpr (RAW == 0) {
      float2* dst = b ? buf1 : buf0;
      mbar_expect_tx(&mbar[b], (uint32_t)(BUF * sizeof(float2)));
#pragma unroll
      for (int r = 0; r < L; r += ROWS_PER_BOX)
        tma_load_2d(dst + r * T, &tmap, (int)b0, (int)(a * L + r), &mbar[b]);
    } else {
      unsigned char* dst = b ? raw1 : raw0;
      mbar_expect_tx(&mbar[b], (uint32_t)(L * rp.row_bytes));
#pragma unroll
      for (int r = 0; r < L; r += ROWS_PER_BOX)
        tma_load_2d(dst + (size_t)r * rp.row_bytes, &tmap, (int)(b0 / T) * rp.row_bytes, (int)(a * L + r), &mbar[b]);
    }
  };
  uint32_t tile = blockIdx.x;
  if (tile < ntiles && tid == 0) issue(tile, 0);
  for (uint32_t it = 0; tile < ntiles; tile += gridDim.x, it++) {
    const int b = ONE_RAW ? 0 : (it & 1);
    float2* const sm = (RAW == 0) ? (b ? buf1 : buf0) : buf0;
    const uint32_t nxt = tile + gridDim.x;
    if (!ONE_RAW && nxt < ntiles && tid == 0) issue(nxt, b ^ 1);
    mbar_wait(&mbar[b], ONE_RAW ? (it & 1) : ((it >> 1) & 1));
    float2 v[16];
    int oidx[16];
    const int up = PADX ? u + (u >> 4) : u;  // tile row of slot 0
    float2 wb, r1;                           // inter-sweep twiddle of slot 0 and the ratio between slots
    if constexpr (STWG) {                    // from global memory: issued before the stages to hide the latency
      const uint32_t bb = (tile % btiles) * T + t;
      wb = big_tw_lookup_ldg(stw, btw.q, (uint32_t)u * bb);
      r1 = big_tw_lookup_ldg(stw, btw.q, (uint32_t)U * bb);
    }
    if constexpr (RAW == 0) {
#pragma unroll
      for (int e = 0; e < 16; e++) v[e] = sm[(u + e * U) * T + t];
      if constexpr (CH) {
        const uint32_t ta = tile / btiles, tb0 = (tile % btiles) * T;
        const float limit = cp.threshold * __ldg(cp.mean);
        if (cp.phase != nullptr) {
          // tabulated phases (block path): T consecutive entries per tile row
          const float* const ph = cp.phase + ((size_t)ta << LOGL) * B + (size_t)u * B + tb0 + t;
          float ang[16];
#pragma unroll
          for (int e = 0; e < 16; e++) ang[e] = __ldg(ph + (size_t)e * U * B);
#pragma unroll
          for (int e = 0; e < 16; e++) v[e] = chirp_point_tab(v[e], ang[e], limit, cp.coef);
        } else {
          double idx = (double)(((size_t)ta << LOGL) * B + (size_t)u * B + tb0 + t);
          const double step = (double)((size_t)U * B);
          double f = fma(cp.df, idx, cp.f_min);
          double r = __drcp_rn(f);
#pragma unroll
          for (int e = 0; e < 16; e++) {
            if (e > 0) {
              idx += step;
              f = fma(cp.df, idx, cp.f_min);
              if (cp.newton == 0) {
                r = __drcp_rn(f);
              } else {
                r = fma(r, fma(-f, r, 1.0), r);
                if (cp.newton > 1) r = fma(r, fma(-f, r, 1.0), r);
              }
            }
            v[e] = chirp_point(v[e], f, r, cp, limit);
          }
        }
      }
    } else if constexpr (RAW == 3) {
      // packed samples: point t of a row occupies bits [2 bits t, 2 bits (t + 1)) counted from the row's MSB
      const int nb = rp.bits, per_byte = 4 / nb, p = t % per_byte;
      const int sh_re = 8 - nb * (2 * p + 1), sh_im = sh_re - nb, mask = (1 << nb) - 1;
      const unsigned char* rawb = (b ? raw1 : raw0) + t / per_byte;
#pragma unroll
      for (int e = 0; e < 16; e++) {
        const unsigned w = rawb[(size_t)(u + e * U) * rp.row_bytes];
        v[e] = make_float2((float)((w >> sh_re) & mask), (float)((w >> sh_im) & mask));
      }
    } else {
      const unsigned char* rawb = (b ? raw1 : raw0) + (size_t)t * rp.G - (size_t)((t & 1) * rp.delta);
#pragma unroll
      for (int e = 0; e < 16; e++) {
        const unsigned char* g = rawb + (size_t)(u + e * U) * rp.row_bytes;
        if (RAW == 1) v[e] = make_float2((float)(int)(signed char)g[rp.o0], (float)(int)(signed char)g[rp.o1]);
        else v[e] = make_float2((float)g[rp.o0], (float)g[rp.o1]);
      }
    }
    if constexpr (ONE_RAW) {
      __syncthreads();  // the raw tile is decoded: the next one may land in its buffer while the stages run
      if (nxt < ntiles && tid == 0) issue(nxt, 0);
    }
    stage_compute16<LOGL, SC::logr(0), 0, FWD, LOGL - SC::logr(0), PADX>(v, u, ltw, oidx);
    if constexpr (RAW == 0) __syncthreads();  // every thread has read the tile before it is overwritten
#pragma unroll
    for (int e = 0; e < 16; e++) sm[oidx[e] * T + t] = v[e];
    __syncthreads();
    if constexpr (S == 3) {
#pragma unroll
      for (int e = 0; e < 16; e++) v[e] = sm[(up + e * UP) * T + t];
      __syncthreads();
      stage_compute16<LOGL, SC::logr(1), SC::logns(1), FWD, LOGL - SC::logns(1) - SC::logr(1), PADX>(v, u, ltw, oidx);
#pragma unroll
      for (int e = 0; e < 16; e++) sm[oidx[e] * T + t] = v[e];
      __syncthreads();
    }
#pragma unroll
    for (int e = 0; e < 16; e++) v[e] = sm[(up + e * UP) * T + t];
    stage_compute16<LOGL, SC::logr(S - 1), SC::logns(S - 1), FWD>(v, u, ltw, oidx);
    {
      // store k = u + e*U of column b0 + t, times W_{L*B}^{k (b0 + t)} = wb * r1^e; the sixteen powers
      // are formed as hi[e >> 2] * lo[e & 3] (products of at most three table values deep)
      const uint32_t a = tile / btiles, b0 = (tile % btiles) * T;
      if constexpr (!STWG) {
        const uint32_t bb = b0 + t;
        wb = big_tw_lookup(stw, btw.q, (uint32_t)u * bb);
        r1 = big_tw_lookup(stw, btw.q, (uint32_t)U * bb);
      }
      if (!FWD) {
        wb.y = -wb.y;
        r1.y = -r1.y;
      }
      const float2 r2 = c_sqr(r1), r3 = c_mul(r2, r1), r4 = c_sqr(r2), r8 = c_sqr(r4), r12 = c_mul(r8, r4);
      const float2 hi1 = c_mul(wb, r4), hi2 = c_mul(wb, r8), hi3 = c_mul(wb, r12);
      float2* o = out + ((size_t)a << LOGL) * B + b0 + (size_t)u * B + t;
#pragma unroll
      for (int e = 0; e < 16; e++) {
        const float2 h = (e >> 2) == 0 ? wb : ((e >> 2) == 1 ? hi1 : ((e >> 2) == 2 ? hi2 : hi3));
        const float2 w = (e & 3) == 0 ? h : c_mul(h, (e & 3) == 1 ? r1 : ((e & 3) == 2 ? r2 : r3));
        o[(size_t)e * U * B] = c_mul(v[e], w);
      }
    }
    __syncthreads();  // buffer b (and the exchange buffer) may be refilled from the next iteration on
  }
}

template <int LOGL, int T, bool FWD, int RAW = 0, bool CH = false>
__global__ void __launch_bounds__(col16_threads<LOGL, T>::value, CH ? 2 : col16_threads<LOGL, T>::min_blocks)
    fft_col16_tma_kernel(const __grid_constant__ tensor_map_blob tmap, float2* __restrict__ out, size_t B,
                         uint32_t btiles, uint32_t ntiles, big_twiddle btw, const float2* __restrict__ tw,
                         raw_params rp, row_chirp_params cp) {
  col16_body<LOGL, T, FWD, RAW, CH>(&tmap, out, B, btiles, ntiles, btw, tw, rp, cp);
}

// the first sweep of the sweep-order R2C route (srtb_b200.cu, r2c_sweep_order): 2^11-point raw columns, T = 8, one
// raw tile buffer (raw16_smem), one CTA of 1024 threads per SM
template <int RAW>
__global__ void __launch_bounds__(col16_threads<11, 8>::value, 1)
    r2c_raw_col2048_kernel(const __grid_constant__ tensor_map_blob tmap, float2* __restrict__ out, size_t B,
                           uint32_t btiles, uint32_t ntiles, big_twiddle btw, const float2* __restrict__ tw,
                           raw_params rp) {
  col16_body<11, 8, true, RAW, false>(&tmap, out, B, btiles, ntiles, btw, tw, rp, row_chirp_params{});
}

// Transposing last pass, persistent: input rows [beta][k1][rest][L] as a 3-D tensor (L, S, L1*batch);
// a tile = T consecutive k1 at fixed (beta, rest) = ONE 3-D TMA box (L, 1, T) landing as [t][L].
// Stage 0 runs in the row mapping on that buffer, then the rotated column layout takes over and the
// results leave in natural order: out[beta*n + k1 + L1*rest + A*k].
template <int LOGL, int T, bool FWD>
__global__ void __launch_bounds__(pass_threads<LOGL, T>::value, pass_threads<LOGL, T>::min_blocks)
    fft_trans_tma_kernel(const __grid_constant__ tensor_map_blob tmap, float2* __restrict__ out, uint32_t A,
                         uint32_t S_, uint32_t L1, uint32_t k1tiles, uint32_t ntiles,
                         const float2* __restrict__ tw, float2* __restrict__ tile_stats) {
  using SC = sched<LOGL>;
  using LAY = tile_layout<LOGL, T, MODE_TRANS>;
  constexpr int L = 1 << LOGL, U = L / 8, S = SC::S, BUF = tile_tma_smem<LOGL, T>::BUF;
  __shared__ float2 stat_sm[2][32];
  extern __shared__ __align__(128) unsigned char smraw[];
  float2* const buf0 = reinterpret_cast<float2*>(smraw);
  float2* const buf1 = buf0 + BUF;
  uint64_t* const mbar = reinterpret_cast<uint64_t*>(buf1 + BUF);
  float2* const ltw = reinterpret_cast<float2*>(smraw + tile_tma_smem<LOGL, T>::data_bytes + 128);
  const int tid = threadIdx.x;
  for (int i = tid; i < L; i += blockDim.x) ltw[i] = __ldg(&tw[i]);
  const int t0 = tid / U, u0 = tid % U;  // stage 0: lanes along the FFT index (rows are contiguous)
  const int t1 = tid % T, u1 = tid / T;  // later stages and the store: lanes along t
  if (tid == 0) {
    mbar_init(&mbar[0], 1);
    mbar_init(&mbar[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  constexpr int COLS_PER_BOX = (L < 256) ? L : 256;
  auto issue = [&](uint32_t tl, int b) {
    const uint32_t k1t = tl % k1tiles, r = tl / k1tiles;
    const uint32_t rest = r % S_, beta = r / S_;
    float2* dst = b ? buf1 : buf0;
    fence_proxy_async();
    mbar_expect_tx(&mbar[b], (uint32_t)(BUF * sizeof(float2)));
    if (L <= 256) {
      tma_load_3d(dst, &tmap, 0, (int)rest, (int)(beta * L1 + k1t * T), &mbar[b]);
    } else {
      // box inner dimension is capped at 256 elements: one box per 256-column slab and per row
      for (int tt = 0; tt < T; tt++)
        for (int c = 0; c < L; c += COLS_PER_BOX)
          tma_load_3d(dst + tt * L + c, &tmap, c, (int)rest, (int)(beta * L1 + k1t * T + tt), &mbar[b]);
    }
  };
  uint32_t tile = blockIdx.x;
  if (tile < ntiles && tid == 0) issue(tile, 0);
  for (uint32_t it = 0; tile < ntiles; tile += gridDim.x, it++) {
    const int b = it & 1;
    float2* const sm = b ? buf1 : buf0;
    const uint32_t nxt = tile + gridDim.x;
    if (nxt < ntiles && tid == 0) issue(nxt, b ^ 1);
    mbar_wait(&mbar[b], (it >> 1) & 1);
    float2 v[8];
    int oidx[8];
#pragma unroll
    for (int e = 0; e < 8; e++) v[e] = sm[t0 * L + u0 + e * U];
    stage_compute<LOGL, SC::logr(0), 0, FWD>(v, u0, tw, oidx);
    __syncthreads();
#pragma unroll
    for (int e = 0; e < 8; e++) sm[LAY::at(oidx[e], t0)] = v[e];
    __syncthreads();
    if constexpr (S >= 3) {
#pragma unroll
      for (int e = 0; e < 8; e++) v[e] = sm[LAY::at(u1 + e * U, t1)];
      __syncthreads();
      stage_compute<LOGL, SC::logr(1), SC::logns(1), FWD, true, LOGL - SC::logns(1) - SC::logr(1), false>(v, u1, ltw, oidx);
#pragma unroll
      for (int e = 0; e < 8; e++) sm[LAY::at(oidx[e], t1)] = v[e];
      __syncthreads();
    }
    if constexpr (S >= 4) {
#pragma unroll
      for (int e = 0; e < 8; e++) v[e] = sm[LAY::at(u1 + e * U, t1)];
      __syncthreads();
      stage_compute<LOGL, SC::logr(2), SC::logns(2), FWD, true, LOGL - SC::logns(2) - SC::logr(2), false>(v, u1, ltw, oidx);
#pragma unroll
      for (int e = 0; e < 8; e++) sm[LAY::at(oidx[e], t1)] = v[e];
      __syncthreads();
    }
#pragma unroll
    for (int e = 0; e < 8; e++) v[e] = sm[LAY::at(u1 + e * U, t1)];
    stage_compute<LOGL, SC::logr(S - 1), SC::logns(S - 1), FWD, true, LOGL - SC::logns(S - 1) - SC::logr(S - 1), false>(v, u1, ltw, oidx);
    {
      const uint32_t k1t = tile % k1tiles, r = tile / k1tiles;
      const uint32_t rest = r % S_, beta = r / S_;
      float2* o = out + (((size_t)beta * A) << LOGL) + (size_t)k1t * T + (size_t)L1 * rest + t1 + (size_t)A * u1;
#pragma unroll
      for (int e = 0; e < 8; e++) o[(size_t)A * e * U] = v[e];
    }
    if (tile_stats) {
      float s2 = 0.f, s4 = 0.f;
#pragma unroll
      for (int e = 0; e < 8; e++) {
        const float p = v[e].x * v[e].x + v[e].y * v[e].y;
        s2 += p;
        s4 += p * p;
      }
#pragma unroll
      for (int o2 = 16; o2 > 0; o2 >>= 1) {
        s2 += __shfl_xor_sync(0xffffffffu, s2, o2);
        s4 += __shfl_xor_sync(0xffffffffu, s4, o2);
      }
      if ((tid & 31) == 0) stat_sm[it & 1][tid >> 5] = make_float2(s2, s4);
    }
    __syncthreads();
    if (tile_stats && tid == 0) {
      float2 a = stat_sm[it & 1][0];
      for (int w = 1; w < (int)(blockDim.x >> 5); w++) {
        a.x += stat_sm[it & 1][w].x;
        a.y += stat_sm[it & 1][w].y;
      }
      tile_stats[tile] = a;
    }
  }
}


// Four-sweep transforms (n = L1*L2*L3*L): the rows of the last sweep are stored as [k1][k2][k3] (k3 fastest),
// natural order needs k1 + L1*(k2 + L2*k3): swap the two digits of `rest` (rest_inner = L3; 0 or 1 = no swap).
__device__ __forceinline__ uint32_t rest_digit_swap(uint32_t rest, uint32_t S_, uint32_t rest_inner) {
  if (rest_inner <= 1) return rest;
  return rest / rest_inner + (S_ / rest_inner) * (rest % rest_inner);
}

// Sixteen-points-per-thread transposing last sweep (L = 128 as 16 x 8, L = 256 as 16 x 16), T = 16 rows
// per tile: stage 0 in the row mapping on the TMA buffer, one exchange through the rotated layout,
// stage 1 in the column mapping, results straight from registers in natural order.
template <int LOGL, int T, bool FWD>
__global__ void __launch_bounds__(T * ((1 << LOGL) / 16), 768 / (T * ((1 << LOGL) / 16)))
    fft_trans16_tma_kernel(const __grid_constant__ tensor_map_blob tmap, float2* __restrict__ out, uint32_t A,
                           uint32_t S_, uint32_t L1, uint32_t k1tiles, uint32_t ntiles,
                           const float2* __restrict__ tw, uint32_t rest_inner, float2* __restrict__ tile_stats) {
  using SC = sched16<LOGL>;
  static_assert(SC::S == 2 && T == 16 && LOGL <= 8, "two radix stages, sixteen rows per tile");
  constexpr int L = 1 << LOGL, U = L / 16, BUF = tile_tma_smem<LOGL, T>::BUF;
  __shared__ float2 stat_sm[2][32];
  extern __shared__ __align__(128) unsigned char smraw[];
  float2* const buf0 = reinterpret_cast<float2*>(smraw);
  float2* const buf1 = buf0 + BUF;
  uint64_t* const mbar = reinterpret_cast<uint64_t*>(buf1 + BUF);
  float2* const ltw = reinterpret_cast<float2*>(smraw + tile_tma_smem<LOGL, T>::data_bytes + 128);
  const int tid = threadIdx.x;
  for (int i = tid; i < L; i += blockDim.x) ltw[i] = __ldg(&tw[i]);
  const int t0 = tid / U, u0 = tid % U;  // stage 0: lanes along the FFT index (rows are contiguous)
  const int t1 = tid % T, u1 = tid / T;  // stage 1 and the store: lanes along t
  auto at = [](int idx, int t) { return idx * T + ((t + (idx >> 4)) & (T - 1)); };
  if (tid == 0) {
    mbar_init(&mbar[0], 1);
    mbar_init(&mbar[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  auto issue = [&](uint32_t tl, int b) {
    const uint32_t k1t = tl % k1tiles, r = tl / k1tiles;
    const uint32_t rest = r % S_, beta = r / S_;
    fence_proxy_async();
    mbar_expect_tx(&mbar[b], (uint32_t)(BUF * sizeof(float2)));
    tma_load_3d(b ? buf1 : buf0, &tmap, 0, (int)rest, (int)(beta * L1 + k1t * T), &mbar[b]);
  };
  uint32_t tile = blockIdx.x;
  if (tile < ntiles && tid == 0) issue(tile, 0);
  for (uint32_t it = 0; tile < ntiles; tile += gridDim.x, it++) {
    const int b = it & 1;
    float2* const sm = b ? buf1 : buf0;
    const uint32_t nxt = tile + gridDim.x;
    if (nxt < ntiles && tid == 0) issue(nxt, b ^ 1);
    mbar_wait(&mbar[b], (it >> 1) & 1);
    float2 v[16];
    int oidx[16];
#pragma unroll
    for (int e = 0; e < 16; e++) v[e] = sm[t0 * L + u0 + e * U];
    stage_compute16<LOGL, SC::logr(0), 0, FWD>(v, u0, ltw, oidx);
    __syncthreads();
#pragma unroll
    for (int e = 0; e < 16; e++) sm[at(oidx[e], t0)] = v[e];
    __syncthreads();
#pragma unroll
    for (int e = 0; e < 16; e++) v[e] = sm[at(u1 + e * U, t1)];
    stage_compute16<LOGL, SC::logr(1), SC::logns(1), FWD>(v, u1, ltw, oidx);
    {
      const uint32_t k1t = tile % k1tiles, r = tile / k1tiles;
      const uint32_t rest = r % S_, beta = r / S_;
      const uint32_t prest = rest_digit_swap(rest, S_, rest_inner);
      float2* o = out + (((size_t)beta * A) << LOGL) + (size_t)k1t * T + (size_t)L1 * prest + t1 + (size_t)A * u1;
#pragma unroll
      for (int e = 0; e < 16; e++) o[(size_t)A * e * U] = v[e];
    }
    if (tile_stats) {
      // spectral-kurtosis statistics of this tile (sum |y|^2, sum |y|^4) for the row decision taken after the sweep
      // (rfi_mitigation.hpp:292-341): warp partials now, folded by thread 0 after the tile's closing barrier
      float s2 = 0.f, s4 = 0.f;
#pragma unroll
      for (int e = 0; e < 16; e++) {
        const float p = v[e].x * v[e].x + v[e].y * v[e].y;
        s2 += p;
        s4 += p * p;
      }
#pragma unroll
      for (int o2 = 16; o2 > 0; o2 >>= 1) {
        s2 += __shfl_xor_sync(0xffffffffu, s2, o2);
        s4 += __shfl_xor_sync(0xffffffffu, s4, o2);
      }
      if ((tid & 31) == 0) stat_sm[it & 1][tid >> 5] = make_float2(s2, s4);
    }
    __syncthreads();
    if (tile_stats && tid == 0) {
      float2 a = stat_sm[it & 1][0];
      for (int w = 1; w < (int)(blockDim.x >> 5); w++) {
        a.x += stat_sm[it & 1][w].x;
        a.y += stat_sm[it & 1][w].y;
      }
      tile_stats[tile] = a;
    }
  }
}


// ---------------------------------------------------------------------------------
// Last pass of the packed real transform with the R2C split fused in (process_block only).
// H = FFT_M(x_even + i x_odd) is produced by this pass in natural order; the split
//   X_k = F + G w,  X_{M-k} = conj(F - G w),  F = (H_k + conj H_{M-k})/2,  G = -i (H_k - conj H_{M-k})/2
// needs H_k and H_{M-k} together. With k = k1 + L1*rest + A*kk (A = L1*S) the mirror of
// (k1, rest, kk) is (L1 - k1, S-1-rest, L-1-kk) for k1 >= 1, so a CTA transforms a primary tile of T
// consecutive k1 AND its mirror tile (two TMA boxes), exchanges the 2T*L results through shared
// memory once and writes final X for both. Column k1 = 0 mirrors onto itself with a carry; it is
// stored raw here and finished by r2c_col0_fixup_kernel, which also completes the mean of |X|^2.
// ---------------------------------------------------------------------------------
template <int LOGL, int T>
struct trans_r2c_smem {
  static constexpr int L = 1 << LOGL;
  static constexpr int BUF = 2 * T * (L + 1);  // [2T][L] raw / exchange, reused as [2T][L+1] results
  static constexpr size_t bytes = 2 * (size_t)BUF * sizeof(float2) + 128 + 2 * (size_t)L * sizeof(float2);
};

__device__ __forceinline__ float2 r2c_split_twiddle(size_t k, size_t M) {
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

template <int LOGL, int T>
__global__ void __launch_bounds__(2 * pass_threads<LOGL, T>::value)
    fft_trans_r2c_tma_kernel(const __grid_constant__ tensor_map_blob tmap, float2* __restrict__ out, uint32_t A,
                             uint32_t S_, uint32_t L1, uint32_t tiles_per_rest, uint32_t ntiles,
                             const float2* __restrict__ tw, double* __restrict__ partial) {
  constexpr bool FWD = true;
  constexpr int T2 = 2 * T;
  using SC = sched<LOGL>;
  using LAY = tile_layout<LOGL, T2, MODE_TRANS>;
  constexpr int L = 1 << LOGL, U = L / 8, S = SC::S, BUF = trans_r2c_smem<LOGL, T>::BUF, LP = L + 1;
  extern __shared__ __align__(128) unsigned char smraw[];
  float2* const buf0 = reinterpret_cast<float2*>(smraw);
  float2* const buf1 = buf0 + BUF;
  uint64_t* const mbar = reinterpret_cast<uint64_t*>(buf1 + BUF);
  float2* const ltw = reinterpret_cast<float2*>(smraw + 2 * (size_t)BUF * sizeof(float2) + 128);
  float2* const htw = ltw + L;  // e^{-i pi kk / L}
  __shared__ double red[32];
  const int tid = threadIdx.x;
  for (int i = tid; i < L; i += blockDim.x) {
    ltw[i] = __ldg(&tw[i]);
    float sn, cs;
    sincospif(-(float)i / (float)L, &sn, &cs);
    htw[i] = make_float2(cs, sn);
  }
  const int t0 = tid / U, u0 = tid % U;    // stage 0: lanes along the FFT index
  const int t1 = tid % T2, u1 = tid / T2;  // later stages: lanes along the 2T sequences
  if (tid == 0) {
    mbar_init(&mbar[0], 1);
    mbar_init(&mbar[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  const size_t M = (size_t)A << LOGL;
  auto issue = [&](uint32_t tl, int b) {
    const uint32_t tau = tl % tiles_per_rest, rest = tl / tiles_per_rest;
    const uint32_t k10 = tau * T;
    float2* dst = b ? buf1 : buf0;
    fence_proxy_async();
    mbar_expect_tx(&mbar[b], (uint32_t)(T2 * L * sizeof(float2)));
    tma_load_3d(dst, &tmap, 0, (int)rest, (int)k10, &mbar[b]);                                          // primary
    tma_load_3d(dst + T * L, &tmap, 0, (int)(S_ - 1 - rest), (int)(L1 - k10 - (T - 1)), &mbar[b]);      // mirror
  };
  float acc = 0.f;
  uint32_t tile = blockIdx.x;
  if (tile < ntiles && tid == 0) issue(tile, 0);
  for (uint32_t it = 0; tile < ntiles; tile += gridDim.x, it++) {
    const int b = it & 1;
    float2* const sm = b ? buf1 : buf0;
    const uint32_t nxt = tile + gridDim.x;
    if (nxt < ntiles && tid == 0) issue(nxt, b ^ 1);
    mbar_wait(&mbar[b], (it >> 1) & 1);
    float2 v[8];
    int oidx[8];
#pragma unroll
    for (int e = 0; e < 8; e++) v[e] = sm[t0 * L + u0 + e * U];
    stage_compute<LOGL, SC::logr(0), 0, FWD>(v, u0, tw, oidx);
    __syncthreads();
#pragma unroll
    for (int e = 0; e < 8; e++) sm[LAY::at(oidx[e], t0)] = v[e];
    __syncthreads();
    if constexpr (S >= 3) {
#pragma unroll
      for (int e = 0; e < 8; e++) v[e] = sm[LAY::at(u1 + e * U, t1)];
      __syncthreads();
      stage_compute<LOGL, SC::logr(1), SC::logns(1), FWD, true, LOGL - SC::logns(1) - SC::logr(1), false>(v, u1, ltw, oidx);
#pragma unroll
      for (int e = 0; e < 8; e++) sm[LAY::at(oidx[e], t1)] = v[e];
      __syncthreads();
    }
#pragma unroll
    for (int e = 0; e < 8; e++) v[e] = sm[LAY::at(u1 + e * U, t1)];
    stage_compute<LOGL, SC::logr(S - 1), SC::logns(S - 1), FWD, true, LOGL - SC::logns(S - 1) - SC::logr(S - 1), false>(v, u1, ltw, oidx);
    __syncthreads();  // exchange buffer fully read: reuse it as the [2T][L+1] result array
#pragma unroll
    for (int e = 0; e < 8; e++) sm[t1 * LP + u1 + e * U] = v[e];
    __syncthreads();
    {
      const uint32_t tau = tile % tiles_per_rest, rest = tile / tiles_per_rest;
      const uint32_t k10 = tau * T;
      const bool last_tile = (tau == tiles_per_rest - 1);  // k10 == L1/2: only its slot 0 is new work
      // thread (u1, t1): primary slot t = t1 % T, output indices kk = u1 + e*U for e in [4*(t1/T), 4*(t1/T)+4)
      const int t = t1 % T, e0 = 4 * (t1 / T);
      const uint32_t k1 = k10 + t;
      // w(gk) = e^{-i pi gk / M} with gk = (k1 + L1 rest) + A kk and A/M = 1/L:
      // one sincospi per thread for the tile-constant factor, e^{-i pi kk / L} from a 2L-point table
      const float2 wbase = r2c_split_twiddle((size_t)k1 + (size_t)L1 * rest, M);
#pragma unroll
      for (int e = e0; e < e0 + 4; e++) {
        const int kk = u1 + e * U;
        const float2 hk = sm[t * LP + kk];
        const float2 hm = sm[(T2 - 1 - t) * LP + (L - 1 - kk)];
        const size_t gk = (size_t)k1 + (size_t)L1 * rest + (size_t)A * kk;
        // the self-mirrored column k1 = L1/2 is reached from both (rest, kk) and (S-1-rest, L-1-kk):
        // take each pair once so the result does not depend on which CTA writes last
        const bool self_dup = last_tile && (rest > S_ - 1 - rest || (rest == S_ - 1 - rest && 2 * kk >= L));
        if (k1 == 0) {
          out[gk] = hk;  // column 0: raw H, finished by the fix-up kernel
        } else if (!(last_tile && t > 0) && !self_dup) {
          const float2 F = make_float2(0.5f * (hk.x + hm.x), 0.5f * (hk.y - hm.y));
          const float2 G = make_float2(0.5f * (hk.y + hm.y), -0.5f * (hk.x - hm.x));
          const float2 w = c_mul(wbase, htw[kk]);
          const float2 gw = make_float2(G.x * w.x - G.y * w.y, G.x * w.y + G.y * w.x);
          const float2 xk = make_float2(F.x + gw.x, F.y + gw.y);
          const float2 xm = make_float2(F.x - gw.x, -(F.y - gw.y));
          out[gk] = xk;
          out[M - gk] = xm;
          acc += (xk.x * xk.x + xk.y * xk.y) + (xm.x * xm.x + xm.y * xm.y);
        }
      }
    }
    __syncthreads();  // result array consumed: the buffer may be refilled from the next iteration on
  }
  // per-CTA partial of sum |X|^2 (completed by the fix-up kernel)
  double s = (double)acc;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((tid & 31) == 0) red[tid >> 5] = s;
  __syncthreads();
  if (tid == 0) {
    double a = 0.0;
    for (int w = 0; w < (int)(blockDim.x + 31) / 32; w++) a += red[w];
    partial[blockIdx.x] = a;
  }
}

// Sixteen-points-per-thread form of the fused last pass + split (L = 256 as 16 x 16, L = 128 as 16 x 8):
// one exchange between the two stages, then the [2T][L+1] result array; same tiles, mirror rule and
// results (up to fp32 rounding) as fft_trans_r2c_tma_kernel.
template <int LOGL, int T>
__global__ void __launch_bounds__(2 * T * ((1 << LOGL) / 16), 3)
    fft_trans_r2c16_tma_kernel(const __grid_constant__ tensor_map_blob tmap, float2* __restrict__ out, uint32_t A,
                               uint32_t S_, uint32_t L1, uint32_t tiles_per_rest, uint32_t ntiles,
                               const float2* __restrict__ tw, double* __restrict__ partial, uint32_t rest_inner) {
  constexpr bool FWD = true;
  constexpr int T2 = 2 * T;
  using SC = sched16<LOGL>;
  static_assert(SC::S == 2 && T2 == 16, "two radix stages, sixteen sequences per tile");
  constexpr int L = 1 << LOGL, U = L / 16, BUF = trans_r2c_smem<LOGL, T>::BUF, LP = L + 1;
  extern __shared__ __align__(128) unsigned char smraw[];
  float2* const buf0 = reinterpret_cast<float2*>(smraw);
  float2* const buf1 = buf0 + BUF;
  uint64_t* const mbar = reinterpret_cast<uint64_t*>(buf1 + BUF);
  float2* const ltw = reinterpret_cast<float2*>(smraw + 2 * (size_t)BUF * sizeof(float2) + 128);
  float2* const htw = ltw + L;  // e^{-i pi kk / L}
  __shared__ double red[32];
  const int tid = threadIdx.x;
  for (int i = tid; i < L; i += blockDim.x) {
    ltw[i] = __ldg(&tw[i]);
    float sn, cs;
    sincospif(-(float)i / (float)L, &sn, &cs);
    htw[i] = make_float2(cs, sn);
  }
  const int t0 = tid / U, u0 = tid % U;    // stage 0: lanes along the FFT index
  const int t1 = tid % T2, u1 = tid / T2;  // stage 1: lanes along the 2T sequences
  // exchange layout: column rotated by idx >> 4 so both mappings are conflict-free
  auto at = [](int idx, int t) { return idx * T2 + ((t + (idx >> 4)) & (T2 - 1)); };
  if (tid == 0) {
    mbar_init(&mbar[0], 1);
    mbar_init(&mbar[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();
  const size_t M = (size_t)A << LOGL;
  auto issue = [&](uint32_t tl, int b) {
    const uint32_t tau = tl % tiles_per_rest, rest = tl / tiles_per_rest;
    const uint32_t k10 = tau * T;
    float2* dst = b ? buf1 : buf0;
    fence_proxy_async();
    mbar_expect_tx(&mbar[b], (uint32_t)(T2 * L * sizeof(float2)));
    tma_load_3d(dst, &tmap, 0, (int)rest, (int)k10, &mbar[b]);                                          // primary
    tma_load_3d(dst + T * L, &tmap, 0, (int)(S_ - 1 - rest), (int)(L1 - k10 - (T - 1)), &mbar[b]);      // mirror
  };
  float acc = 0.f;
  uint32_t tile = blockIdx.x;
  if (tile < ntiles && tid == 0) issue(tile, 0);
  for (uint32_t it = 0; tile < ntiles; tile += gridDim.x, it++) {
    const int b = it & 1;
    float2* const sm = b ? buf1 : buf0;
    const uint32_t nxt = tile + gridDim.x;
    if (nxt < ntiles && tid == 0) issue(nxt, b ^ 1);
    mbar_wait(&mbar[b], (it >> 1) & 1);
    float2 v[16];
    int oidx[16];
#pragma unroll
    for (int e = 0; e < 16; e++) v[e] = sm[t0 * L + u0 + e * U];
    stage_compute16<LOGL, SC::logr(0), 0, FWD>(v, u0, ltw, oidx);
    __syncthreads();
#pragma unroll
    for (int e = 0; e < 16; e++) sm[at(oidx[e], t0)] = v[e];
    __syncthreads();
#pragma unroll
    for (int e = 0; e < 16; e++) v[e] = sm[at(u1 + e * U, t1)];
    stage_compute16<LOGL, SC::logr(1), SC::logns(1), FWD>(v, u1, ltw, oidx);
    __syncthreads();  // exchange buffer fully read: reuse it as the [2T][L+1] result array
#pragma unroll
    for (int e = 0; e < 16; e++) sm[t1 * LP + u1 + e * U] = v[e];
    __syncthreads();
    {
      const uint32_t tau = tile % tiles_per_rest, rest = tile / tiles_per_rest;
      const uint32_t k10 = tau * T;
      const bool last_tile = (tau == tiles_per_rest - 1);  // k10 == L1/2: only its slot 0 is new work
      // split mapping (its own; the results sit in shared memory): a warp takes primary slots t = 0..7 and the four
      // residues kk mod 16 = {c, c+8, c+1, c+9}, in that order over its four groups of eight lanes: 8-byte shared
      // loads are served per HALF warp, and with rows LP = L + 1 apart t + kk then covers every value mod 16 exactly
      // once in each half — one wavefront per half for the element and for its mirror (the former (u1, t1) mapping
      // needed two); kk = residue + 16 e, warps 4..7 (L = 256) taking e = 8..15
      const int lane = tid & 31, wsp = tid >> 5;
      const int t = lane & 7, kl = 2 * (wsp & 3) + (lane >> 4) + 8 * ((lane >> 3) & 1), e0 = 8 * (wsp >> 2);
      const uint32_t k1 = k10 + t;
      const uint32_t prest = rest_digit_swap(rest, S_, rest_inner);
      const float2 wbase = r2c_split_twiddle((size_t)k1 + (size_t)L1 * prest, M);
#pragma unroll
      for (int e = e0; e < e0 + 8; e++) {
        const int kk = kl + e * 16;
        const float2 hk = sm[t * LP + kk];
        const float2 hm = sm[(T2 - 1 - t) * LP + (L - 1 - kk)];
        const size_t gk = (size_t)k1 + (size_t)L1 * prest + (size_t)A * kk;
        const bool self_dup = last_tile && (rest > S_ - 1 - rest || (rest == S_ - 1 - rest && 2 * kk >= L));
        if (k1 == 0) {
          out[gk] = hk;  // column 0: raw H, finished by the fix-up kernel
        } else if (!(last_tile && t > 0) && !self_dup) {
          const float2 F = make_float2(0.5f * (hk.x + hm.x), 0.5f * (hk.y - hm.y));
          const float2 G = make_float2(0.5f * (hk.y + hm.y), -0.5f * (hk.x - hm.x));
          const float2 w = c_mul(wbase, htw[kk]);
          const float2 gw = make_float2(G.x * w.x - G.y * w.y, G.x * w.y + G.y * w.x);
          const float2 xk = make_float2(F.x + gw.x, F.y + gw.y);
          const float2 xm = make_float2(F.x - gw.x, -(F.y - gw.y));
          out[gk] = xk;
          out[M - gk] = xm;
          acc += (xk.x * xk.x + xk.y * xk.y) + (xm.x * xm.x + xm.y * xm.y);
        }
      }
    }
    __syncthreads();  // result array consumed: the buffer may be refilled from the next iteration on
  }
  double s = (double)acc;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((tid & 31) == 0) red[tid >> 5] = s;
  __syncthreads();
  if (tid == 0) {
    double a = 0.0;
    for (int w = 0; w < (int)(blockDim.x + 31) / 32; w++) a += red[w];
    partial[blockIdx.x] = a;
  }
}

// column k1 = 0 of the fused split (indices that are multiples of L1, mirror = M - index), the Nyquist
// bin, and the final mean of |X_k|^2 over k < M. Pairs are dealt grid-stride; the last CTA to finish adds the
// partials of the fused pass and of this kernel in index order.
__global__ void __launch_bounds__(256) r2c_col0_fixup_kernel(float2* __restrict__ H, size_t M, size_t L1,
                                                              double* __restrict__ partial, unsigned nparts,
                                                              unsigned* __restrict__ ticket,
                                                              float* __restrict__ mean_out) {
  __shared__ double red[8];
  __shared__ bool last;
  pdl_launch_dependents();
  pdl_wait();
  const size_t n = M / L1;  // column length; pairs j <-> n - j
  double acc = 0.0;
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j <= n / 2; j += (size_t)gridDim.x * blockDim.x) {
    const size_t k = j * L1;
    const float2 hk = H[k];
    const float2 hm = (k == 0) ? hk : H[M - k];
    const float2 F = make_float2(0.5f * (hk.x + hm.x), 0.5f * (hk.y - hm.y));
    const float2 G = make_float2(0.5f * (hk.y + hm.y), -0.5f * (hk.x - hm.x));
    const float2 w = r2c_split_twiddle(k, M);
    const float2 gw = make_float2(G.x * w.x - G.y * w.y, G.x * w.y + G.y * w.x);
    const float2 xk = make_float2(F.x + gw.x, F.y + gw.y);
    const float2 xm = make_float2(F.x - gw.x, -(F.y - gw.y));
    H[k] = xk;
    H[M - k] = xm;
    const float wm = (k == 0 || 2 * k == M) ? 0.f : 1.f;
    acc += (double)((xk.x * xk.x + xk.y * xk.y) + wm * (xm.x * xm.x + xm.y * xm.y));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0;
    for (int w = 0; w < 8; w++) a += red[w];
    partial[nparts + blockIdx.x] = a;
    __threadfence();
    last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
    if (last) __threadfence();  // one acquiring fence (a fence per warp serialises: ~1 us each)
  }
  __syncthreads();
  if (last) {
    double a = 0.0;
    for (unsigned i = threadIdx.x; i < nparts + gridDim.x; i += blockDim.x) a += partial[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = a;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
      for (int w = 0; w < 8; w++) t += red[w];
      *mean_out = (float)t / (float)M;
      *ticket = 0;
    }
  }
}

}  // namespace srtb_b200
