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
  // the R2C row sweep (SRC = 2) adds one double per thread (its group's Σ|X|^2 over the rows, handed over by whichever
  // CTA summed it) and the mbarrier on which the partner CTA releases half buffer B
  static constexpr size_t bytes_r2c = bytes + NT * sizeof(double) + 8;
  // the sweep-order load (SRC = 1) lands 128-byte-swizzled tensor boxes, whose destinations must be 1024-byte aligned:
  // half buffers rounded up to 1 KiB, and 1 KiB more to align the base of the dynamic shared memory
  static constexpr int HALF_SW = (HALF + 127) / 128 * 128;
  static constexpr size_t bytes_sw = bytes + 3 * (size_t)(HALF_SW - HALF) * sizeof(float2) + 1024;
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

// ---- distributed shared memory of a two-CTA cluster (the R2C row sweep reads its partner row's spectrum)
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t dsmem_addr(const void* p, unsigned rank) {
  uint32_t a;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(smem_u32(p)), "r"(rank));
  return a;
}
__device__ __forceinline__ float4 ld_dsmem_f4(uint32_t a) {
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a) : "memory");
  return v;
}
// arrive on an mbarrier of a CTA of the cluster without waiting for this thread's earlier stores
__device__ __forceinline__ void mbar_arrive_dsmem_relaxed(uint32_t a) {
  asm volatile("mbarrier.arrive.relaxed.cluster.shared::cluster.b64 _, [%0];" ::"r"(a) : "memory");
}
__device__ __forceinline__ double ld_dsmem_f64(uint32_t a) {
  double v;
  asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void st_dsmem_f64(uint32_t a, double v) {
  asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(a), "d"(v) : "memory");
}

// R2C split of bin k = k1 + P k2 from Z[k] and Z[M - k] (w = e^{-i pi k / M}):
//   X[k] = (Z[k] + conj Z[M-k]) / 2 - i w (Z[k] - conj Z[M-k]) / 2, the expression of fft_trans_r2c16_tma_kernel
__device__ __forceinline__ float2 r2c_split_point(float2 hk, float2 hm, float2 w) {
  const float2 F = make_float2(0.5f * (hk.x + hm.x), 0.5f * (hk.y - hm.y));
  const float2 G = make_float2(0.5f * (hk.y + hm.y), -0.5f * (hk.x - hm.x));
  const float2 gw = make_float2(G.x * w.x - G.y * w.y, G.x * w.y + G.y * w.x);
  return make_float2(F.x + gw.x, F.y + gw.y);
}

// the R2C row sweep (SRC = 2): rows of the [P][L] scratch, Σ|X|^2 partials per CTA, mean over M = P L bins
struct r2c_rows_params {
  double* partial;
  unsigned* ticket;
  float* mean;
};

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
//   4 = two and two, 2 = a correctly rounded reciprocal for every bin (widely spaced bins of short test blocks, and the
//   sweep-order load, SRC = 1), 5 = the phase table's angles (natural-order rows only)
// SRC: where the rows come from and what is stored.
//   0 = rows of `in` (natural order), natural-order rows to `out`;
//   1 = channel `row` of a spectrum left channel-blocked by SRC = 2 (bin k = k1 + P k2 at (k2 >> 3) L + 8 k1 + (k2 & 7),
//       P = L / 8): one contiguous range of L elements laid out [k1][k2 & 7], fetched through `tmap` as 8 boxes of 128
//       lines x 128 bytes (a quarter of a half buffer each, one mbarrier each), 128-byte swizzled: 16-byte piece q of
//       line t lands at piece q ^ (t & 7). Chunk d0 of the channel is column d0 >> 1, rows from (P / 2) (d0 & 1):
//       buffer A holds rows k1 < P / 2, buffer B the rest, and stage 0 gathers butterfly j from rows j and j + P / 2
//       before it stores the standard layout (tools/proto_r2c_sweep_order.py);
//   2 = the R2C row sweep, run as clusters of two CTAs: nrows = P rows of the scratch `in`, the cluster's CTAs take
//       rows i and P - i (cluster 0: rows 0 and P / 2, each its own mirror), transform them forward and store the split
//       spectrum X[k1 + P k2] channel-blocked to `out`, each CTA splitting half of the pair's mirror pairs for both rows
//       and reading their mirror halves through distributed shared memory.
// The body is shared by three entry points: fft_bigrow_kernel (SRC = 0) and the two kernels of the sweep-order R2C
// route below it.
template <int LOGL, bool FWD, bool SK, int CHIRP, int SRC>
__device__ __forceinline__ void bigrow_body(const float2* __restrict__ in, float2* __restrict__ out, unsigned nrows,
                                            const float2* __restrict__ tabs, const row_sk_params& skp,
                                            const row_chirp_params& cp, const tensor_map_blob* tmap,
                                            const r2c_rows_params& rr) {
  static_assert(SRC == 0 || (LOGL == 14 && ((SRC == 1 && !FWD && SK && CHIRP == 2) || (SRC == 2 && FWD && !SK && CHIRP == 0))),
                "sweep-order routes: rows of 2^14");
  using C = bigrow<LOGL>;
  constexpr int L = C::L, R3 = C::R3, B1 = C::B1, B2 = C::B2, S1 = C::S1, S2 = C::S2, NT = C::NT, NW = C::NW;
  constexpr int HALF = (SRC == 1) ? C::HALF_SW : C::HALF;  // stride of the half buffers, elements
  constexpr size_t off_tab = 3 * (size_t)HALF * sizeof(float2);
  constexpr size_t off_mbar = off_tab + (size_t)C::TABN * sizeof(float2);
  constexpr size_t off_red = off_mbar + 24 * 8;
  extern __shared__ __align__(128) unsigned char smraw[];
  unsigned char* const sm = (SRC == 1) ? smraw + ((0u - smem_u32(smraw)) & 1023u) : smraw;
  float2* const hbuf = reinterpret_cast<float2*>(sm);  // three half-row buffers
  float2* const T0 = reinterpret_cast<float2*>(sm + off_tab);
  float2* const T1 = T0 + B1;
  float2* const T2 = T1 + 15 * B2;
  uint64_t* const mbar = reinterpret_cast<uint64_t*>(sm + off_mbar);  // [3 buffers][8 chunks]
  float* const red = reinterpret_cast<float*>(sm + off_red);  // [2 slots][s2 | s4][32]
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  // SRC = 1, 2: the per-row addresses of stages 1 and 2, of the last stage and of the split come from a thread index
  // read afresh (volatile), so they cost a few integer operations per row instead of registers kept live through the
  // butterflies and, in SRC = 1, the chirp angles (a spill)
  auto tid_row = [&]() -> int {
    if constexpr (SRC != 0) {
      unsigned t;
      asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t));
      return (int)t;
    } else {
      return tid;
    }
  };

  // SRC = 2: per thread t of a one-group-per-thread split, its group's Σ|X|^2 over the rows; the mbarrier on which the
  // CTA holding the mirror row signals that it has read this CTA's half buffer B. Their addresses are formed afresh at
  // each use (volatile), not kept live through the butterflies (a spill)
  auto gsum_at = [&]() {
    unsigned o;
    asm volatile("mov.u32 %0, %1;" : "=r"(o) : "n"((unsigned)C::bytes));
    return reinterpret_cast<double*>(sm + o);
  };
  auto bfree_at = [&]() { return reinterpret_cast<uint64_t*>(gsum_at() + NT); };
  for (int i = tid; i < C::TABN; i += NT) T0[i] = __ldg(&tabs[i]);
  if (tid < 24) mbar_init(&mbar[tid], 1);
  if constexpr (SRC == 2) {
    gsum_at()[tid] = 0.0;
    if (tid == 0) mbar_init(bfree_at(), 1);
  }
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
    if constexpr (SRC == 1) {
      if (lane < 4) {  // rows k1 = (P / 2) which + 256 lane .. + 255 of channel `row`: 128 lines of 128 bytes
        mbar_expect_tx(&mbar[hb * 8 + lane], (uint32_t)(256 * 8 * sizeof(float2)));
        tma_load_2d(hbuf + hb * HALF + lane * 2048, tmap, 0, (int)(row * (L / 16) + (L / 32) * which + 128 * lane),
                    &mbar[hb * 8 + lane]);
      }
    } else {
      const int c = tid_row() & 31;  // the lane
      if (c < 8) {
        mbar_expect_tx(&mbar[hb * 8 + c], (uint32_t)(B1 * sizeof(float2)));
        bulk_g2s(hbuf + hb * HALF + c * S1, in + (size_t)row * L + (size_t)(which * 8 + c) * B1,
                 (uint32_t)(B1 * sizeof(float2)), &mbar[hb * 8 + c]);
      }
    }
  };

  // CHIRP = 5: one 128-byte line of the row's phases per thread (L * 4 bytes = NT lines), asked into L2 ahead of use
  auto prefetch_phase = [&](unsigned r) {
    if constexpr (CHIRP == 5)
      asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(cp.phase + (size_t)r * L) + (size_t)tid * 128));
  };
  // the row of iteration it: SRC = 2 walks pairs (i, P - i) cluster by cluster, the others rows blockIdx.x + it gridDim.x
  const unsigned crank = blockIdx.x & 1;
  auto row_of = [&](unsigned it) -> unsigned {
    if constexpr (SRC == 2) {
      const unsigned i = (blockIdx.x >> 1) + it * (gridDim.x >> 1);
      return i == 0 ? crank * (nrows / 2) : (crank ? nrows - i : i);
    } else {
      return blockIdx.x + it * gridDim.x;
    }
  };
  // SRC = 2: rows 0 and P / 2 are their own mirrors; the CTA holding the mirror row of `r` (the partner, or this one)
  auto self_paired = [&](unsigned r) { return r == 0 || 2 * r == nrows; };
  auto mirror_rank = [&](unsigned r) { return self_paired(r) ? crank : (crank ^ 1); };
  // SRC = 2: thread t of the split holds group t & ~8 (pd0 < 8) of a one-group-per-thread map, whose thread indices
  // the Σ|X|^2 fold keeps; its mirror group (15 - pd0, 15 - pd1, 1 - sel) is that map's thread NT - 1 - (t & ~8)
  auto mirror_slot = [](int t) { return NT - 1 - (t & ~8); };
  auto live = [&](unsigned it) -> bool {
    if constexpr (SRC == 2) return (blockIdx.x >> 1) + it * (gridDim.x >> 1) < nrows / 2;
    else return row_of(it) < nrows;
  };
  if (live(0)) prefetch_phase(row_of(0));  // the table is a constant of the run: no dependency to wait for
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
  if constexpr (SRC == 2) {
    // e^{-i pi i2 / 64}, i2 = 0..15: the split twiddle's factor along the output digit d2 (k2 = .. + 256 d2)
    if (tid < 16) {
      float sn, cs;
      sincospif(-(float)tid / 64.f, &sn, &cs);
      reinterpret_cast<float2*>(red)[tid] = make_float2(cs, sn);
    }
    __syncthreads();
  }
  double psum = 0.0;  // SRC = 2: Σ|X|^2 of the thread's own group (threads h = 1 of the split)
  if (wid == 0) {
    if (live(0)) {
      issue_half(row_of(0), 0, 0);
      issue_half(row_of(0), 1, 1);
    }
    if (live(1)) issue_half(row_of(1), 0, 2);
  }
  for (unsigned it = 0; live(it); it++) {
    const unsigned row = row_of(it);
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
      if constexpr (SRC == 1) {
        // rows j, j + 1 of each half are line tid, 128 contiguous bytes: eight 16-byte pieces (columns 2 (p & 3),
        // 2 (p & 3) + 1 of row j + (p >> 2)). The swizzled load left piece p at p ^ (tid & 7), so a quarter warp reading
        // piece p touches eight distinct bank groups. Piece p of half h holds k1 = (P / 2) h + j + (p >> 2) at columns
        // k2' = 2 (p & 3) + e, e = 0, 1: bin k1 + P (8 row + k2') = row L + k1 + P k2'. Its phase is evaluated exactly
        // (chirp_angle, the phase table's expression) rather than read from a table (2 bytes per sample). The angles
        // do not depend on the data, so each half's sixteen are formed before its wait: half B of this row was issued
        // only at the end of the previous row, and its wait is where the fp64 work can hide.
        const int rot = tid & 7, box = tid >> 7;
        const double bin0 = (double)((size_t)row * L + j);  // below 2^25: every bin below is an exact double
#pragma unroll
        for (int h = 0; h < 2; h++) {
          float ang[16];
#pragma unroll
          for (int p = 0; p < 8; p++)
#pragma unroll
            for (int e = 0; e < 2; e++)
              ang[2 * p + e] = chirp_angle(bin0 + (double)((L / 16) * h + (p >> 2) + (L / 8) * (2 * (p & 3) + e)),
                                           cp.f_min, cp.df, cp.inv_fc, cp.f_c, cp.ddm);
          // the angles are formed before the wait, not sunk past it by the compiler
#pragma unroll
          for (int i = 0; i < 16; i++) asm volatile("" : "+f"(ang[i]));
          mbar_wait(&mbar[(h ? hB : hA) * 8 + box], h ? parB : parA);
          const float4* const src = reinterpret_cast<const float4*>((h ? bufB : bufA) + 8 * j);
#pragma unroll
          for (int p = 0; p < 8; p++) {
            const float4 x = src[p ^ rot];
            const int c = 2 * (p & 3);  // columns c, c + 1 -> d0 = 2 c + h, 2 c + 2 + h
            const float2 y0 = chirp_point_tab(make_float2(x.x, x.y), ang[2 * p], limit, cp.coef);
            const float2 y1 = chirp_point_tab(make_float2(x.z, x.w), ang[2 * p + 1], limit, cp.coef);
            if (p < 4) {
              a[2 * c + h] = y0;
              a[2 * c + 2 + h] = y1;
            } else {
              b[2 * c + h] = y0;
              b[2 * c + 2 + h] = y1;
            }
          }
        }
        // every thread has gathered its rows before the layout is rewritten; the barrier comes before the butterflies
        // so that their stores can follow the twiddles one by one (after them, all 64 results would be live at once)
        __syncthreads();
      } else if constexpr (CHIRP == 5) {
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
      if constexpr (CHIRP != 5 && SRC != 1) {
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
      const int t = tid_row();
      const int d0 = t / (B2 / 2), jp = t % (B2 / 2);
      bigrow_stage_table<FWD, S2, B2>(half_of(d0) + 2 * jp, T1 + 2 * jp);
    }
    __syncthreads();
    // ---- stage 2: block (d0, d1), butterflies over d2 (stride R3), pair of [0, R3); lanes vary d0
    {
      const int t = tid_row();
      const int d0 = t & 15, rest = t >> 4, jp = rest % (R3 / 2), d1 = rest / (R3 / 2);
      bigrow_stage_table<FWD, R3, R3>(half_of(d0) + d1 * S2 + 2 * jp, T2 + 2 * jp);
    }
    __syncthreads();
    // ---- last stage, pass 1: radix R3 on R3 contiguous elements, in place; row statistics for SK
    float s2 = 0.f, s4 = 0.f;
    if constexpr (R3 == 4) {
      const int t = tid_row();
#pragma unroll
      for (int g = 0; g < 8; g++) {
        const int rest = (t >> 4) + (NT / 16) * g;  // lanes vary d0; (d1, d2) = rest
        float2* const p = half_of(t & 15) + (rest >> 4) * S2 + (rest & 15) * 4;
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
    if constexpr (SRC == 2) cluster_sync_all();  // both rows of the pair are transformed
    else __syncthreads();
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
    if (live(it + 1)) prefetch_phase(row_of(it + 1));
    if constexpr (SRC == 2) {
      // ---- R2C split and channel-blocked store of the pair: X[k1 + P k2] of row k1 = row and of its mirror row prow
      // (P - row; row itself for rows 0 and P / 2, which the partner CTA does not share). X[k] and X[M - k] come from
      // the same two inputs Z[k], Z[M - k], so each pair is read once and split once for both bins: this CTA takes the
      // pairs whose own bin has d0 < 8 (its half buffer A, local) and reads their mirrors, d0 >= 8, from half buffer B
      // of the mirror row (remote: 64 KiB per row). The groups are those of a one-group-per-thread map, thread
      // (pd0, pd1, sel) holding 32 bins: k2 = pd0 + 16 pd1 + 256 i2 + 4096 d3, d3 = 2 sel, 2 sel + 1. A thread here
      // takes group (pd0 < 8, pd1, sel) at i2 = 0..7 (h = 0) or 15..8 (h = 1), and the mirror group
      // (15 - pd0, 15 - pd1, 1 - sel) at 15 - i2 (tools/proto_r2c_sweep_order.py, paired_split). For k1 != 0 the mirror
      // of k2 is L - 1 - k2: every digit complemented, (d0, d1, d2, d3) -> (15 - d0, 15 - d1, 15 - d2, 3 - d3), so the
      // mirror group's 16-byte pair at 15 - i2 holds the two mirrors with its halves swapped.
      const unsigned prow = self_paired(row) ? row : nrows - row, prank = mirror_rank(row);
      const int t = tid_row(), lane = t & 31, wid = t >> 5;
      const int pd0 = lane & 7, h = (lane >> 3) & 1, pd1 = ((wid & 7) << 1) | (lane >> 4), sel = wid >> 3;
      const float2* const base = bufA + pd0 * S1 + pd1 * S2 + 2 * sel;
      const uint32_t mbase = dsmem_addr(bufB + (7 - pd0) * S1 + (15 - pd1) * S2 + 2 * (1 - sel), prank);
      const int kb = pd0 + 16 * pd1 + 4096 * (2 * sel);                   // k2 of d2 = 0, d3 = 2 sel
      const int kbm = (15 - pd0) + 16 * (15 - pd1) + 4096 * (2 * (1 - sel));  // the same of the mirror group
      float2 wb, wbm;  // e^{-i pi (k1 + P kb) / M} of each group; both fractions are exact in fp32
      {
        float sn, cs;
        sincospif(-((float)row / ((float)nrows * (float)L) + (float)kb / (float)L), &sn, &cs);
        wb = make_float2(cs, sn);
        sincospif(-((float)prow / ((float)nrows * (float)L) + (float)kbm / (float)L), &sn, &cs);
        wbm = make_float2(cs, sn);
      }
      const float2* const htw = reinterpret_cast<const float2*>(red);
      auto pos = [&](int k) {  // shared-memory position of natural-order k2 (pass 2's digit map)
        return half_of(k & 15) + ((k >> 4) & 15) * S2 + ((k >> 8) & 15) * R3 + (k >> 12);
      };
      // X[k1 + P k2] goes to (k2 >> 3) L + 8 k1 + (k2 & 7): channel k2 >> 3 (L = 8 P bins) is one contiguous range,
      // the order of the phase table and of the waterfall kernel's load. Lanes 2m and 2m + 1 hold k2 and k2 + 1 (pd0 even
      // and odd; of the mirror groups, odd and even): they trade halves, and each stores a 16-byte pair, the even one at
      // d3 = 2 sel, the odd one at d3 = 2 sel + 1. Eight lanes store two whole 64-byte pieces; rows 2m and 2m + 1 fill
      // the two halves of each line.
      const unsigned odd = lane & 1;
      const int ks = kb + (int)odd * 4095, ksm = kbm + (int)(odd ^ 1) * 4095;  // k2 of the stored pair's first element
      float2* const o = out + (size_t)(ks >> 3) * L + 8 * (size_t)row + (ks & 7);
      float2* const om = out + (size_t)(ksm >> 3) * L + 8 * (size_t)prow + (ksm & 7);
      auto store_pair = [&](float2* p, unsigned od, float2 x0, float2 x1) {
        const float2 mine = od ? x0 : x1;
        const float2 theirs = make_float2(__shfl_xor_sync(0xffffffffu, mine.x, 1), __shfl_xor_sync(0xffffffffu, mine.y, 1));
        *reinterpret_cast<float4*>(p) = od ? make_float4(theirs.x, theirs.y, x1.x, x1.y) : make_float4(x0.x, x0.y, theirs.x, theirs.y);
      };
      auto norm2 = [](float2 x0, float2 x1) { return (x0.x * x0.x + x0.y * x0.y) + (x1.x * x1.x + x1.y * x1.y); };
      // Σ|X|^2 of each group is the fp32 sum over i2 = 0..15 in that order: h = 0 sums its own group's i2 = 0..7 and
      // h = 1 the mirror group's (15 - i2 ascends as i2 descends); each keeps the other group's eight terms and adds
      // them, i2 ascending, to the partial its lane + 8 hands over
      float seq = 0.f, terms[8];
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const int i2 = h ? 15 - j : j, im = 15 - i2;
        const float4 q = *reinterpret_cast<const float4*>(base + i2 * R3);
        const float4 r = ld_dsmem_f4(mbase + (uint32_t)(im * R3 * sizeof(float2)));
        float2 m0, m1, mm0, mm1;  // the mirrors of q's and of r's two elements
        if (row != 0) {
          m0 = make_float2(r.z, r.w);
          m1 = make_float2(r.x, r.y);
          mm0 = make_float2(q.z, q.w);
          mm1 = make_float2(q.x, q.y);
        } else {  // row 0 pairs k2 with (L - k2) mod L, in this CTA
          const int k0 = kb + 256 * i2, km0 = kbm + 256 * im;
          m0 = *pos((L - k0) & (L - 1));
          m1 = *pos((L - k0 - 4096) & (L - 1));
          mm0 = *pos((L - km0) & (L - 1));
          mm1 = *pos((L - km0 - 4096) & (L - 1));
        }
        const float2 w0 = c_mul(wb, htw[i2]);
        const float2 w1 = c_mul(w0, make_float2(0.70710678118654752440f, -0.70710678118654752440f));  // k2 + L / 4
        const float2 v0 = c_mul(wbm, htw[im]);
        const float2 v1 = c_mul(v0, make_float2(0.70710678118654752440f, -0.70710678118654752440f));
        const float2 x0 = r2c_split_point(make_float2(q.x, q.y), m0, w0);
        const float2 x1 = r2c_split_point(make_float2(q.z, q.w), m1, w1);
        const float2 y0 = r2c_split_point(make_float2(r.x, r.y), mm0, v0);
        const float2 y1 = r2c_split_point(make_float2(r.z, r.w), mm1, v1);
        store_pair(o + (size_t)i2 * (32 * L), odd, x0, x1);
        store_pair(om + (size_t)im * (32 * L), odd ^ 1, y0, y1);
        const float tx = norm2(x0, x1), ty = norm2(y0, y1);
        seq += h ? ty : tx;
        terms[j] = h ? tx : ty;
      }
      float gs = __shfl_xor_sync(0xffffffffu, seq, 8);
#pragma unroll
      for (int j = 7; j >= 0; j--) gs += terms[j];
      // Σ over rows in row order, in double, of each group: h = 1 adds its own group's; h = 0 the mirror group's, which
      // belongs to the partner from its first row on. Only cluster 0 has rows 0 and P / 2, at it = 0: there the mirror
      // group is this CTA's own, so its partial goes to gsum here, and the partner thread continues that sum from it
      if (h || !self_paired(row)) {
        if (!h && it == (blockIdx.x < 2 ? 1u : 0u)) psum = ld_dsmem_f64(dsmem_addr(gsum_at() + mirror_slot(t), prank));
        psum += (double)gs;
      } else {
        gsum_at()[mirror_slot(t)] = (double)gs;
      }
    } else {
    // ---- pass 2: natural-order store. lane -> (d0, d1 bit 0): 32 consecutive output indices per instruction
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
    // the row's buffers are free: second half of the next row, first half of the one after
    __syncthreads();
    if constexpr (SRC == 2) {
      // The split read buffer A only here and buffer B only in the CTA of the mirror row (here too for rows 0 and P / 2),
      // so each is released on its own, and no cluster barrier waits for the split's stores. A, which takes the next
      // row's second half (stage 0 needs it first), is free after the barrier above. B is free once the mirror row's
      // CTA has arrived on bfree, which it does after its own barrier above: its remote reads of B have returned their
      // values by then (they were consumed by the split), and the copy into B is issued only after the wait. Each CTA
      // gets one arrive per row (from its partner, or from itself for rows 0 and P / 2), so bfree completes phase `it`
      // in row `it`; the partner cannot arrive for row it + 1 before both CTAs pass the cluster barrier of row it + 1.
      if (wid == 0) {
        if (live(it + 1)) issue_half(row_of(it + 1), 1, hA);  // B of row it + 1 is A of row it
        if (lane == 0) mbar_arrive_dsmem_relaxed(dsmem_addr(bfree_at(), mirror_rank(row)));
        if (live(it + 2)) {
          mbar_wait(bfree_at(), it & 1);
          issue_half(row_of(it + 2), 0, hB);  // A of row it + 2 is B of row it
        }
      }
    } else if (wid == 0) {
      if (live(it + 1)) issue_half(row_of(it + 1), 1, hA);  // B of row it + 1 is A of row it
      if (live(it + 2)) issue_half(row_of(it + 2), 0, hB);  // A of row it + 2 is B of row it
    }
  }
  if constexpr (SRC == 2) {
    // Σ|X|^2: the h = 1 threads store their own groups' sums, the h = 0 threads hand the mirror groups' sums to the
    // partner (not after a CTA with only a self-paired row: its mirror group's sum is already in gsum); the cluster
    // barrier makes those visible and keeps both CTAs' shared memory alive past the last remote access. Then thread t holds group t's sum, as a one-group-per-thread split would: per-CTA
    // partial, then the last CTA folds the partials in index order (as r2c_col0_fixup_kernel does)
    double* const gsum = gsum_at();
    if ((tid >> 3) & 1) gsum[tid & ~8] = psum;
    else if (blockIdx.x >= 2 || live(1)) st_dsmem_f64(dsmem_addr(gsum + mirror_slot(tid), crank ^ 1), psum);
    cluster_sync_all();
    double* const redd = reinterpret_cast<double*>(red + 64);
    unsigned* const last = reinterpret_cast<unsigned*>(red + 96);
    double v = gsum[tid];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) redd[wid] = v;
    __syncthreads();
    if (tid == 0) {
      double a = 0.0;
      for (int w = 0; w < NW; w++) a += redd[w];
      rr.partial[blockIdx.x] = a;
      __threadfence();
      *last = (atomicAdd(rr.ticket, 1u) == gridDim.x - 1) ? 1u : 0u;
      if (*last) __threadfence();
    }
    __syncthreads();
    if (*last && wid == 0) {
      double a = 0.0;
      for (unsigned i = lane; i < gridDim.x; i += 32) a += __ldcg(&rr.partial[i]);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
      if (lane == 0) {
        *rr.mean = (float)a / ((float)nrows * (float)L);
        *rr.ticket = 0;
      }
    }
  }
}

template <int LOGL, bool FWD, bool SK, int CHIRP>
__global__ void __launch_bounds__(bigrow<LOGL>::NT, bigrow<LOGL>::CTAS)
    fft_bigrow_kernel(const float2* __restrict__ in, float2* __restrict__ out, unsigned nrows,
                      const float2* __restrict__ tabs, row_sk_params skp, row_chirp_params cp) {
  bigrow_body<LOGL, FWD, SK, CHIRP, 0>(in, out, nrows, tabs, skp, cp, nullptr, r2c_rows_params{});
}

// the sweep-order R2C route of 2^25-point blocks with rows of 2^14 (srtb_b200.cu, r2c_sweep_order): the paired row
// sweep with the split (clusters of two CTAs, from the [P][L] scratch z to the channel-blocked spectrum) ...
__global__ void __launch_bounds__(bigrow<14>::NT, 1)
    r2c_rows_split_kernel(const float2* __restrict__ z, float2* __restrict__ out, unsigned nrows,
                          const float2* __restrict__ tabs, r2c_rows_params rr) {
  bigrow_body<14, true, false, 0, 2>(z, out, nrows, tabs, row_sk_params{}, row_chirp_params{}, nullptr, rr);
}

// ... and the whole-row waterfall kernel reading channel `row` of that spectrum through a swizzling tensor map
__global__ void __launch_bounds__(bigrow<14>::NT, 1)
    waterfall_sweep_order_kernel(const float2* __restrict__ in, float2* __restrict__ out, unsigned nrows,
                                 const float2* __restrict__ tabs, row_sk_params skp, row_chirp_params cp,
                                 const __grid_constant__ tensor_map_blob tmap) {
  bigrow_body<14, false, true, 2, 1>(in, out, nrows, tabs, skp, cp, &tmap, r2c_rows_params{});
}

}  // namespace srtb_b200
