// fft_bigrow.cuh — one-kernel waterfall for long channel rows (L = 2^13, 2^14): a whole row lives in ONE
// CTA's shared memory (64 / 128 KiB), so the chain
//   rfi_mitigation_s1 (zap + normalise)  -> dedisperse chirp -> watfft (backward C2C) -> rfi_mitigation_s2 (SK)
//   -> first stage of signal_detect's column sums
// touches HBM exactly twice (read the spectrum row, write the dynamic-spectrum row). Reference operators:
//   userspace/include/srtb/pipeline/rfi_mitigation_pipe.hpp:66-79, coherent_dedispersion.hpp:133-150,223-237,
//   pipeline/fft_pipe.hpp:313-371, spectrum/rfi_mitigation.hpp:292-341, pipeline/signal_detect_pipe.hpp:296-316.
// (The BASELINE "J1644 shape" has L = Nc / C = 2^25 / 2^11 = 2^14.)
//
// Algorithm (index algebra prototyped and checked against numpy in tools/proto_bigrow.py):
//   * in-place decimation-in-frequency, radices 16 x 16 x 16 x R3 (R3 = L / 4096 = 2 or 4); natural order in,
//     digit-reversed order in shared memory, natural order restored by the final store;
//   * a thread owns TWO adjacent butterflies per stage (32 points) and moves them with 16-byte shared-memory
//     accesses (one LDS.128 / STS.128 per two points, addresses base + i * stride: no per-access integer work);
//   * the sixteen chunks of a row (d0 = 0..15, B1 = L/16 elements each) are stored S1 = B1 + 2 elements apart: the
//     chunk stride is odd in 16-byte units, so lanes that differ in d0 never meet in a bank group, and every other
//     access pattern runs over contiguous pairs — all conflict free, while each chunk stays ONE contiguous TMA copy;
//   * rows arrive by TMA bulk copies (cp.async.bulk, one per chunk: sixteen 8 KiB copies per 2^14-point row), each
//     signalled on its own mbarrier. Shared memory holds THREE half-row buffers that
//     rotate: while row r is transformed in two of them, the first half of row r + 1 lands in the third, and its
//     second half follows into the buffer row r frees first — stage 0 consumes chunk i while chunks i + 1.. arrive;
//   * the detector's column sums (one accumulator per time sample, 64 KiB for 2^14) fit neither in shared memory
//     (three half rows and the tables take 209 KiB of the 227 KiB a block may have) nor in registers (the
//     butterflies use all 128 a thread gets at 512 threads): every thread owns 32 cells of its CTA's partial row in
//     global memory, read and written back once per row with an L2 evict-last policy, so the row stays in L2
//     (grid x ts_count x 4 bytes: 8 MiB per lane on 132 SMs, against 50 MB) while the spectrum streams past it;
//   * twiddles: stage 0 from W_L^j by repeated multiplication, stages 1 and 2 from small shared-memory tables;
//   * the chirp phase is evaluated in fp64 like the reference; 1/f comes from one correctly rounded reciprocal per
//     thread and Newton steps from the neighbouring bin: one step when (B1*df/f)^2 <= 2^-52 (the reciprocal is then
//     good to an ulp, the accuracy of the reference's own fp64 division chain), two when the fourth power keeps the
//     phase error below 1e-9 cycles, otherwise the exact reciprocal of every bin; the fractional
//     part by the round-to-nearest trick (e^{-2 pi i k} only needs k mod 1), sin/cos from the SFU on [-pi, pi].
#pragma once
#include "fft_engine.cuh"

namespace srtb_b200 {

template <int LOGL>
struct bigrow {
  static_assert(LOGL == 13 || LOGL == 14, "whole-row kernel: L = 8192 or 16384");
  static constexpr int L = 1 << LOGL;
  static constexpr int R3 = L / 4096;
  static constexpr int B1 = L / 16, B2 = L / 256;
  static constexpr int S2 = B2, S1 = B1 + 2;  // chunks of B1 elements, contiguous inside, two elements apart
  static constexpr int HALF = 8 * S1;       // half a padded row (chunks d0 = 0..7 or 8..15), elements
  static constexpr int NT = L / 32;         // threads: 32 points each
  static constexpr int NW = NT / 32;
  static constexpr int CTAS = (LOGL == 13) ? 2 : 1;
  static constexpr int TABN = B1 + 15 * B2 + 15 * R3;  // W_L^j | W_B1^{i j} [15][B2] | W_B2^{i j} [15][R3]
  static constexpr size_t off_tab = 3 * (size_t)HALF * sizeof(float2);
  static constexpr size_t off_mbar = off_tab + (size_t)TABN * sizeof(float2);
  static constexpr size_t off_red = off_mbar + 24 * 8;   // 3 buffers x 8 chunk barriers
  static constexpr size_t bytes = off_red + 4 * 32 * sizeof(float);
};

// ---- column-sum cells in global memory, kept in L2 across the rows a CTA adds into them
__device__ __forceinline__ uint64_t l2_evict_last_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ float ld_l2_keep(const float* a, uint64_t pol) {
  float v;
  asm volatile("ld.global.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(a), "l"(pol));
  return v;
}
__device__ __forceinline__ void st_l2_keep(float* a, float v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.f32 [%0], %1, %2;" ::"l"(a), "f"(v), "l"(pol) : "memory");
}

// a[i] *= w^i, i = 1..15 (powers at most four multiplications deep)
__device__ __forceinline__ void bigrow_twiddle_powers(float2 (&a)[16], const float2 w1) {
  const float2 w2 = c_sqr(w1), w3 = c_mul(w2, w1), w4 = c_sqr(w2);
  a[1] = c_mul(a[1], w1);
  a[2] = c_mul(a[2], w2);
  a[3] = c_mul(a[3], w3);
  a[4] = c_mul(a[4], w4);
  const float2 w5 = c_mul(w4, w1), w6 = c_sqr(w3), w7 = c_mul(w4, w3), w8 = c_sqr(w4);
  a[5] = c_mul(a[5], w5);
  a[6] = c_mul(a[6], w6);
  a[7] = c_mul(a[7], w7);
  a[8] = c_mul(a[8], w8);
  a[9] = c_mul(a[9], c_mul(w8, w1));
  a[10] = c_mul(a[10], c_sqr(w5));
  a[11] = c_mul(a[11], c_mul(w8, w3));
  a[12] = c_mul(a[12], c_sqr(w6));
  a[13] = c_mul(a[13], c_mul(w8, w5));
  a[14] = c_mul(a[14], c_sqr(w7));
  a[15] = c_mul(a[15], c_mul(w8, w7));
}

// one radix-16 DIF stage on two adjacent butterflies: elements base + i*STRIDE (16-byte pairs), twiddles
// W^{i j} for the pair (j, j + 1) from a table laid out [15][TB] (row i - 1, column j)
template <bool FWD, int STRIDE, int TB>
__device__ __forceinline__ void bigrow_stage_table(float2* __restrict__ p, const float2* __restrict__ tab) {
  float2 a[16], b[16];
#pragma unroll
  for (int i = 0; i < 16; i++) {
    const float4 q = *reinterpret_cast<const float4*>(p + i * STRIDE);
    a[i] = make_float2(q.x, q.y);
    b[i] = make_float2(q.z, q.w);
  }
  dft16<FWD>(a);
  dft16<FWD>(b);
  *reinterpret_cast<float4*>(p) = make_float4(a[0].x, a[0].y, b[0].x, b[0].y);
#pragma unroll
  for (int i = 1; i < 16; i++) {
    const float4 w = *reinterpret_cast<const float4*>(tab + (i - 1) * TB);
    const float2 ya = c_mul(a[i], make_float2(w.x, w.y)), yb = c_mul(b[i], make_float2(w.z, w.w));
    *reinterpret_cast<float4*>(p + i * STRIDE) = make_float4(ya.x, ya.y, yb.x, yb.y);
  }
}

// CHIRP: 0 = plain transform; otherwise s1 + chirp on load, 1/f of successive bins by Newton steps from the neighbour:
//   1 = one step along a butterfly's inputs (B1 bins apart) and one to the adjacent bin, 3 = two and one,
//   4 = two and two, 2 = a correctly rounded reciprocal for every bin (widely spaced bins of short test blocks)
template <int LOGL, bool FWD, bool SK, int CHIRP>
__global__ void __launch_bounds__(bigrow<LOGL>::NT, bigrow<LOGL>::CTAS)
    fft_bigrow_kernel(const float2* __restrict__ in, float2* __restrict__ out, unsigned nrows,
                      const float2* __restrict__ tabs, row_sk_params skp, row_chirp_params cp) {
  using C = bigrow<LOGL>;
  constexpr int L = C::L, R3 = C::R3, B1 = C::B1, B2 = C::B2, S1 = C::S1, S2 = C::S2, NT = C::NT, NW = C::NW;
  constexpr int HALF = C::HALF;
  extern __shared__ __align__(128) unsigned char smraw[];
  float2* const hbuf = reinterpret_cast<float2*>(smraw);  // three half-row buffers
  float2* const T0 = reinterpret_cast<float2*>(smraw + C::off_tab);
  float2* const T1 = T0 + B1;
  float2* const T2 = T1 + 15 * B2;
  uint64_t* const mbar = reinterpret_cast<uint64_t*>(smraw + C::off_mbar);  // [3 buffers][8 chunks]
  float* const red = reinterpret_cast<float*>(smraw + C::off_red);  // [2 slots][s2 | s4][32]
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;

  for (int i = tid; i < C::TABN; i += NT) T0[i] = __ldg(&tabs[i]);
  if (tid < 24) mbar_init(&mbar[tid], 1);
  if (tid == 0) fence_mbar_init();
  __syncthreads();
  // this thread's 32 column-sum cells: time samples kcell + 256 (c >> 1) + 4096 (c & 1) of the CTA's partial row,
  // natural order; cells past ts_count are dropped. Only this thread ever touches them.
  const int kcell = (lane & 15) + 16 * (((wid & 7) << 1) | (lane >> 4)) + 8192 * (wid >> 3);
  float* const cells = skp.partial + (size_t)blockIdx.x * skp.ts_count + kcell;
  auto cell_live = [&](int c) { return (unsigned)(kcell + 256 * (c >> 1) + 4096 * (c & 1)) < skp.ts_count; };
  auto cell = [&](int c) { return cells + 256 * (c >> 1) + 4096 * (c & 1); };
  uint64_t keep_pol = 0;
  if constexpr (SK) keep_pol = l2_evict_last_policy();

  // warp 0, lanes 0..7: fetch half a row (chunks d0 = 8 which .. 8 which + 7) into half buffer hb, one bulk copy per
  // chunk, each signalled on its own mbarrier
  auto issue_half = [&](unsigned row, int which, int hb) {
    fence_proxy_async();
    if (lane < 8) {
      mbar_expect_tx(&mbar[hb * 8 + lane], (uint32_t)(B1 * sizeof(float2)));
      bulk_g2s(hbuf + hb * HALF + lane * S1, in + (size_t)row * L + (size_t)(which * 8 + lane) * B1,
               (uint32_t)(B1 * sizeof(float2)), &mbar[hb * 8 + lane]);
    }
  };

  // CHIRP = 5: one 128-byte line of the row's phases per thread (L * 4 bytes = NT lines), asked into L2 ahead of use
  auto prefetch_phase = [&](unsigned r) {
    if constexpr (CHIRP == 5)
      asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(cp.phase + (size_t)r * L) + (size_t)tid * 128));
  };
  if (blockIdx.x < nrows) prefetch_phase(blockIdx.x);  // the table is a constant of the run: no dependency to wait for
  pdl_launch_dependents();
  pdl_wait();  // tables and barriers were set up while the preceding kernel drained
  if constexpr (SK) {
#pragma unroll
    for (int c = 0; c < 32; c++)
      if (cell_live(c)) st_l2_keep(cell(c), 0.f, keep_pol);
  }
  float limit = 0.f;
  if constexpr (CHIRP) limit = cp.threshold * __ldg(cp.mean);

  // Rotation of the three half buffers: row `it` of this CTA has chunks 0..7 in A = (2 it) % 3 and chunks 8..15 in
  // B = (2 it + 1) % 3; the third buffer receives chunks 0..7 of the next row meanwhile. Buffer A has been filled
  // floor(2 it / 3) times before, B floor((2 it + 1) / 3) times: the mbarrier phase parities.
  unsigned row = blockIdx.x;
  if (wid == 0) {
    if (row < nrows) {
      issue_half(row, 0, 0);
      issue_half(row, 1, 1);
    }
    if (row + gridDim.x < nrows) issue_half(row + gridDim.x, 0, 2);
  }
  for (unsigned it = 0; row < nrows; row += gridDim.x, it++) {
    const int hA = (2 * it) % 3, hB = (2 * it + 1) % 3;
    const unsigned parA = ((2 * it) / 3) & 1, parB = ((2 * it + 1) / 3) & 1;
    float2* const bufA = hbuf + hA * HALF;
    float2* const bufB = hbuf + hB * HALF;
    auto half_of = [&](int d0) { return (d0 < 8 ? bufA : bufB) + (d0 & 7) * S1; };  // first element of chunk d0
    // ---- stage 0: butterflies over d0 (stride S1), pair j = 2 tid, 2 tid + 1 of [0, B1)
    {
      const int j = 2 * tid;
      float2* const pa = bufA + j;
      float2* const pb = bufB + j;
      float2 a[16], b[16];
      if constexpr (CHIRP == 5) {
        // tabulated phases (two adjacent bins per 8-byte load, prefetched into L2 while the previous row was stored):
        // s1 + chirp applied as the pairs are taken out of shared memory, no pass of its own and no fp64
        const float2* const ph = reinterpret_cast<const float2*>(cp.phase + (size_t)row * L + j);
#pragma unroll
        for (int h = 0; h < 2; h++) {
          float2 pq[8];
#pragma unroll
          for (int i = 0; i < 8; i++) pq[i] = __ldg(ph + (size_t)(8 * h + i) * (B1 / 2));
#pragma unroll
          for (int i = 0; i < 8; i++) {
            mbar_wait(&mbar[(h ? hB : hA) * 8 + i], h ? parB : parA);
            const float4 q = *reinterpret_cast<const float4*>((h ? pb : pa) + i * S1);
            a[8 * h + i] = chirp_point_tab(make_float2(q.x, q.y), pq[i].x, limit, cp.coef);
            b[8 * h + i] = chirp_point_tab(make_float2(q.z, q.w), pq[i].y, limit, cp.coef);
          }
        }
      } else if constexpr (CHIRP != 0) {
        // s1 + chirp as a pass of its own over the thread's sixteen pairs, written back in place: no butterfly
        // registers are live yet, so several bins' fp64 phase chains are in flight at once (the thread re-reads only
        // what it wrote itself: no barrier). Chunk i is consumed as soon as it has landed.
        double idx = (double)((size_t)row * L + j);
        double fa = fma(cp.df, idx, cp.f_min);
        double ra = __drcp_rn(fa);
        auto newton = [](double r, double f) { return fma(r, fma(-f, r, 1.0), r); };
        auto refine_far = [&](double r, double f) {   // bin B1 further on
          if constexpr (CHIRP == 2) return __drcp_rn(f);
          r = newton(r, f);
          if constexpr (CHIRP >= 3) r = newton(r, f);
          return r;
        };
        auto refine_near = [&](double r, double f) {  // adjacent bin
          if constexpr (CHIRP == 2) return __drcp_rn(f);
          r = newton(r, f);
          if constexpr (CHIRP == 4) r = newton(r, f);
          return r;
        };
#pragma unroll 4
        for (int i = 0; i < 16; i++) {
          if (i > 0) {
            idx += (double)B1;
            fa = fma(cp.df, idx, cp.f_min);
            ra = refine_far(ra, fa);
          }
          float2* const p = (i < 8 ? pa : pb) + (i & 7) * S1;
          mbar_wait(&mbar[(i < 8 ? hA : hB) * 8 + (i & 7)], i < 8 ? parA : parB);
          const float4 q = *reinterpret_cast<const float4*>(p);
          const float2 ya = chirp_point(make_float2(q.x, q.y), fa, ra, cp, limit);
          const double fb = fma(cp.df, idx + 1.0, cp.f_min);
          const float2 yb = chirp_point(make_float2(q.z, q.w), fb, refine_near(ra, fb), cp, limit);
          *reinterpret_cast<float4*>(p) = make_float4(ya.x, ya.y, yb.x, yb.y);
        }
      }
      if constexpr (CHIRP != 5) {
#pragma unroll
        for (int i = 0; i < 16; i++) {
          if constexpr (CHIRP == 0) mbar_wait(&mbar[(i < 8 ? hA : hB) * 8 + (i & 7)], i < 8 ? parA : parB);
          const float4 q = *reinterpret_cast<const float4*>((i < 8 ? pa : pb) + (i & 7) * S1);
          a[i] = make_float2(q.x, q.y);
          b[i] = make_float2(q.z, q.w);
        }
      }
      dft16<FWD>(a);
      dft16<FWD>(b);
      const float4 w = *reinterpret_cast<const float4*>(T0 + j);
      bigrow_twiddle_powers(a, make_float2(w.x, w.y));
      bigrow_twiddle_powers(b, make_float2(w.z, w.w));
#pragma unroll
      for (int i = 0; i < 16; i++)
        *reinterpret_cast<float4*>((i < 8 ? pa : pb) + (i & 7) * S1) = make_float4(a[i].x, a[i].y, b[i].x, b[i].y);
    }
    __syncthreads();
    // ---- stage 1: block d0, butterflies over d1 (stride S2), pair of [0, B2)
    {
      const int d0 = tid / (B2 / 2), jp = tid % (B2 / 2);
      bigrow_stage_table<FWD, S2, B2>(half_of(d0) + 2 * jp, T1 + 2 * jp);
    }
    __syncthreads();
    // ---- stage 2: block (d0, d1), butterflies over d2 (stride R3), pair of [0, R3); lanes vary d0
    {
      const int d0 = tid & 15, rest = tid >> 4, jp = rest % (R3 / 2), d1 = rest / (R3 / 2);
      bigrow_stage_table<FWD, R3, R3>(half_of(d0) + d1 * S2 + 2 * jp, T2 + 2 * jp);
    }
    __syncthreads();
    // ---- last stage, pass 1: radix R3 on R3 contiguous elements, in place; row statistics for SK
    float s2 = 0.f, s4 = 0.f;
    if constexpr (R3 == 4) {
#pragma unroll
      for (int g = 0; g < 8; g++) {
        const int rest = (tid >> 4) + (NT / 16) * g;  // lanes vary d0; (d1, d2) = rest
        float2* const p = half_of(tid & 15) + (rest >> 4) * S2 + (rest & 15) * 4;
        const float4 q0 = *reinterpret_cast<const float4*>(p), q1 = *reinterpret_cast<const float4*>(p + 2);
        float2 x0 = make_float2(q0.x, q0.y), x1 = make_float2(q0.z, q0.w);
        float2 x2 = make_float2(q1.x, q1.y), x3 = make_float2(q1.z, q1.w);
        dft4<FWD>(x0, x1, x2, x3);
        *reinterpret_cast<float4*>(p) = make_float4(x0.x, x0.y, x1.x, x1.y);
        *reinterpret_cast<float4*>(p + 2) = make_float4(x2.x, x2.y, x3.x, x3.y);
        if constexpr (SK) {
          const float p0 = x0.x * x0.x + x0.y * x0.y, p1 = x1.x * x1.x + x1.y * x1.y;
          const float p2 = x2.x * x2.x + x2.y * x2.y, p3 = x3.x * x3.x + x3.y * x3.y;
          s2 += (p0 + p1) + (p2 + p3);
          s4 += (p0 * p0 + p1 * p1) + (p2 * p2 + p3 * p3);
        }
      }
    } else {
#pragma unroll
      for (int g = 0; g < 16; g++) {
        const int rest = (tid >> 4) + (NT / 16) * g;  // lanes vary d0; (d1, d2) = rest
        float2* const p = half_of(tid & 15) + (rest >> 4) * S2 + (rest & 15) * 2;
        const float4 q = *reinterpret_cast<const float4*>(p);
        const float2 y0 = make_float2(q.x + q.z, q.y + q.w), y1 = make_float2(q.x - q.z, q.y - q.w);
        *reinterpret_cast<float4*>(p) = make_float4(y0.x, y0.y, y1.x, y1.y);
        if constexpr (SK) {
          const float p0 = y0.x * y0.x + y0.y * y0.y, p1 = y1.x * y1.x + y1.y * y1.y;
          s2 += p0 + p1;
          s4 += p0 * p0 + p1 * p1;
        }
      }
    }
    bool zap = false;
    float acc[SK ? 32 : 1];
    if constexpr (SK) {
      // the row's column sums are fetched now, so that L2 latency overlaps the SK reduction below
#pragma unroll
      for (int c = 0; c < 32; c++) acc[c] = cell_live(c) ? ld_l2_keep(cell(c), keep_pol) : 0.f;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
        s4 += __shfl_xor_sync(0xffffffffu, s4, o);
      }
      float* const slot = red + (it & 1) * 64;  // per-warp partials alternate between two slots
      if (lane == 0) {
        slot[wid] = s2;
        slot[32 + wid] = s4;
      }
    }
    __syncthreads();
    if constexpr (SK) {
      // every warp folds the NW per-warp partials with the same fixed shuffle tree
      const float* const slot = red + (it & 1) * 64;
      float a = (lane < NW) ? slot[lane] : 0.f, b = (lane < NW) ? slot[32 + lane] : 0.f;
#pragma unroll
      for (int o = NW / 2; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
      }
      a = __shfl_sync(0xffffffffu, a, 0);
      b = __shfl_sync(0xffffffffu, b, 0);
      const float sk = (float)L * (b / (a * a));
      zap = (sk > skp.thr_hi || sk < skp.thr_lo);  // NaN (all-zero row): untouched (rfi_mitigation.hpp:333-339)
    }
    if (row + gridDim.x < nrows) prefetch_phase(row + gridDim.x);
    // ---- pass 2: natural-order store. lane -> (d0, d1 bit 0): 32 consecutive output indices per instruction
    {
      const int pd0 = lane & 15, pd1 = ((wid & 7) << 1) | (lane >> 4), sel = wid >> 3;
      const float2* const base = half_of(pd0) + pd1 * S2 + 2 * sel;
      float2* const o = out + (size_t)row * L + (pd0 + 16 * pd1 + 4096 * (2 * sel));
      if (zap) {
#pragma unroll
        for (int i2 = 0; i2 < 16; i2++) {
          o[256 * i2] = make_float2(0.f, 0.f);
          o[256 * i2 + 4096] = make_float2(0.f, 0.f);
        }
      } else {
#pragma unroll
        for (int i2 = 0; i2 < 16; i2++) {
          const float4 q = *reinterpret_cast<const float4*>(base + i2 * R3);
          o[256 * i2] = make_float2(q.x, q.y);          // k = d0 + 16 d1 + 256 d2 + 4096 d3, d3 = 2 sel
          o[256 * i2 + 4096] = make_float2(q.z, q.w);   // d3 = 2 sel + 1
          if constexpr (SK) {
            acc[2 * i2] += q.x * q.x + q.y * q.y;
            acc[2 * i2 + 1] += q.z * q.z + q.w * q.w;
          }
        }
        if constexpr (SK) {
#pragma unroll
          for (int c = 0; c < 32; c++)
            if (cell_live(c)) st_l2_keep(cell(c), acc[c], keep_pol);
        }
      }
    }
    __syncthreads();  // the row's buffers are free: second half of the next row, first half of the one after
    if (wid == 0) {
      const unsigned nxt = row + gridDim.x, nxt2 = row + 2 * gridDim.x;
      if (nxt < nrows) issue_half(nxt, 1, hA);     // B of row it + 1 is A of row it
      if (nxt2 < nrows) issue_half(nxt2, 0, hB);   // A of row it + 2 is B of row it
    }
  }
}

}  // namespace srtb_b200
