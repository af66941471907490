// events.cuh — every above-threshold run ("event") of the detector's boxcar series, found on the device
// (srtb_b200_series_events, srtb_b200_incoherent_dm_search_events, srtb_b200_process_block_dm_sweep_events).
//
// An event is a maximal run [begin, end) of one boxcar series v with every v[j] > threshold[b] (count_signal's strict
// comparison), with the smallest index holding the run's largest value and that value over sqrt(variance[b]). The rows
// searched are those the detector headers describe: boxcars b < n_boxcars of every record with detect_enabled, each
// series_length[b] long; the headers are read on the device, where the detector wrote them.
//
// Work split: a row is cut into tiles of EV_TILE samples; one CTA per (tile, boxcar, record), two launches.
//
//   ev_count_kernel  threads read the tile interleaved (coalesced) and reduce it to a summary: the number of runs that
//                    begin in it, and its leading fragment (how many samples from the tile start are above threshold,
//                    their largest value and its first index). The last CTA to finish (ticket) forms the exclusive scan
//                    of the run counts over every tile in (record, boxcar, tile) order, from the stream's running event
//                    count, and advances that count: the scan gives every run its output slot, so the list is in
//                    (stream, trial, boxcar, begin) order and two calls write the same bytes.
//   ev_emit_kernel   CTAs whose tile begins no run exit at once. The others stage the tile in shared memory; a thread
//                    takes EV_PER consecutive samples and reduces them to a leading fragment too. The thread holding a
//                    run's begin follows it through its own samples, then through the following threads' fragments,
//                    then through the following tiles' summaries, so a run that spans many tiles costs its owner
//                    O(EV_PER + EV_THREADS + tiles spanned), never a walk over its samples.
// Events past max_events are counted but not written.
#pragma once
#include <cuda_runtime.h>

#include "ops_kernels.cuh"

namespace srtb_b200 {

constexpr int EV_THREADS = 256;
constexpr int EV_PER = 16;                       // consecutive samples per thread in ev_emit_kernel
constexpr int EV_TILE = EV_THREADS * EV_PER;     // samples per tile

// srtb_b200_event
struct ev_event {
  unsigned long long begin, end, peak_index;
  float snr;
  unsigned trial, boxcar, stream;
};

// a tile's summary: runs beginning in it, and its leading fragment (prefix_len samples from the tile start above
// threshold; prefix_max and its first tile index prefix_arg, when prefix_len > 0)
struct ev_tile {
  unsigned starts;
  unsigned prefix_len;
  float prefix_max;
  unsigned prefix_arg;
};

// the rows of one launch: record y's boxcar b is series + y trial_stride + b boxcar_stride, under header res[y].
// tiles: tiles per row of the longest row the launch may meet; events carry trial trial0 + y and stream `stream`
struct ev_rows {
  const float* series;
  size_t boxcar_stride, trial_stride;
  const detect_dev_result* res;
  unsigned max_nb;
  size_t tiles;
  unsigned trial0, stream;
};

__device__ __forceinline__ bool ev_row(const ev_rows& r, unsigned y, unsigned nb, const float** v, size_t* n,
                                       float* thr, float* var) {
  const detect_dev_result* h = r.res + y;
  if (!h->detect_enabled || (int)nb >= h->n_boxcars) return false;
  *v = r.series + (size_t)y * r.trial_stride + (size_t)nb * r.boxcar_stride;
  *n = h->series_length[nb];
  *thr = h->threshold[nb];
  *var = h->variance[nb];
  return true;
}

// (value, index): the larger value wins, equal values the smaller index; index ~0u = none
__device__ __forceinline__ void ev_better(float& v, unsigned& i, float ov, unsigned oi) {
  if (oi == ~0u) return;
  if (i == ~0u || ov > v || (ov == v && oi < i)) {
    v = ov;
    i = oi;
  }
}

__global__ void __launch_bounds__(EV_THREADS) ev_count_kernel(const ev_rows r, ev_tile* __restrict__ tile,
                                                              unsigned long long* __restrict__ offset,
                                                              unsigned* __restrict__ ticket,
                                                              unsigned long long* __restrict__ count) {
  __shared__ unsigned s_u[EV_THREADS / 32];
  __shared__ float s_v[EV_THREADS / 32];
  __shared__ unsigned s_i[EV_THREADS / 32];
  __shared__ unsigned long long s_w[EV_THREADS / 32];
  __shared__ bool s_last;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const unsigned t = blockIdx.x, nb = blockIdx.y, y = blockIdx.z;
  const size_t k = ((size_t)y * r.max_nb + nb) * r.tiles + t;
  const float* v = nullptr;
  size_t n = 0;
  float thr = 0.f, var = 0.f;
  const bool row = ev_row(r, y, nb, &v, &n, &thr, &var);
  const size_t base = (size_t)t * EV_TILE;
  if (row && base < n) {  // uniform over the CTA
    float x[EV_PER];
    bool prev[EV_PER];
#pragma unroll
    for (int i = 0; i < EV_PER; i++) {
      const size_t j = base + (size_t)i * EV_THREADS + tid;
      x[i] = j < n ? v[j] : NAN;  // NaN: never above
      prev[i] = (j > 0 && j < n) ? (v[j - 1] > thr) : false;
    }
    unsigned starts = 0, below = EV_TILE;
#pragma unroll
    for (int i = 0; i < EV_PER; i++) {
      const bool a = x[i] > thr;
      starts += (a && !prev[i]) ? 1u : 0u;
      if (!a) below = min(below, (unsigned)(i * EV_THREADS + tid));
    }
    // run starts: sum; leading fragment: the first sample not above (min), then the largest value before it
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      starts += __shfl_down_sync(0xffffffffu, starts, o);
      below = min(below, __shfl_down_sync(0xffffffffu, below, o));
    }
    if (lane == 0) {
      s_u[wid] = starts;
      s_i[wid] = below;
    }
    __syncthreads();
    starts = 0;
    below = EV_TILE;
    for (int w = 0; w < EV_THREADS / 32; w++) {
      starts += s_u[w];
      below = min(below, s_i[w]);
    }
    __syncthreads();
    float pm = 0.f;
    unsigned pa = ~0u;
#pragma unroll
    for (int i = 0; i < EV_PER; i++) {
      const unsigned li = (unsigned)(i * EV_THREADS + tid);
      if (li < below) ev_better(pm, pa, x[i], li);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_down_sync(0xffffffffu, pm, o);
      const unsigned oi = __shfl_down_sync(0xffffffffu, pa, o);
      ev_better(pm, pa, ov, oi);
    }
    if (lane == 0) {
      s_v[wid] = pm;
      s_i[wid] = pa;
    }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < EV_THREADS / 32; w++) ev_better(pm, pa, s_v[w], s_i[w]);
      tile[k] = ev_tile{starts, below, below ? pm : 0.f, below ? pa : 0u};
    }
  } else if (tid == 0) {
    tile[k] = ev_tile{0u, 0u, 0.f, 0u};
  }
  // ---- last CTA: exclusive scan of the run counts from the stream's running count. The barrier orders the CTA's
  // store before thread 0's cumulative fence (the pattern of colsum_final_scan_kernel)
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    const unsigned ctas = gridDim.x * gridDim.y * gridDim.z;
    s_last = (atomicAdd(ticket, 1u) == ctas - 1);
    if (s_last) __threadfence();
  }
  __syncthreads();
  if (!s_last) return;
  const size_t nt = (size_t)gridDim.x * gridDim.y * gridDim.z;
  unsigned long long carry = *reinterpret_cast<volatile unsigned long long*>(count);
  constexpr int PER = 8;
  for (size_t b0 = 0; b0 < nt; b0 += (size_t)EV_THREADS * PER) {
    unsigned c[PER];
    unsigned long long local = 0;
#pragma unroll
    for (int e = 0; e < PER; e++) {
      const size_t i = b0 + (size_t)tid * PER + e;
      c[e] = i < nt ? __ldcg(&tile[i].starts) : 0u;
      local += c[e];
    }
    unsigned long long incl = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    if (lane == 31) s_w[wid] = incl;
    __syncthreads();
    unsigned long long before = 0, total = 0;
    for (int w = 0; w < EV_THREADS / 32; w++) {
      if (w < wid) before += s_w[w];
      total += s_w[w];
    }
    unsigned long long run = carry + before + (incl - local);
#pragma unroll
    for (int e = 0; e < PER; e++) {
      const size_t i = b0 + (size_t)tid * PER + e;
      if (i < nt) offset[i] = run;
      run += c[e];
    }
    carry += total;
    __syncthreads();  // s_w consumed
  }
  if (tid == 0) {
    *count = carry;
    *ticket = 0;
  }
}

__global__ void __launch_bounds__(EV_THREADS) ev_emit_kernel(const ev_rows r, const ev_tile* __restrict__ tile,
                                                             const unsigned long long* __restrict__ offset,
                                                             ev_event* __restrict__ out,
                                                             unsigned long long max_events) {
  __shared__ float sv[EV_TILE];
  __shared__ unsigned s_plen[EV_THREADS], s_parg[EV_THREADS];
  __shared__ float s_pmax[EV_THREADS];
  __shared__ unsigned s_w[EV_THREADS / 32];
  __shared__ bool s_before;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const unsigned t = blockIdx.x, nb = blockIdx.y, y = blockIdx.z;
  const size_t row0 = ((size_t)y * r.max_nb + nb) * r.tiles;
  if (tile[row0 + t].starts == 0) return;  // uniform: no run begins here
  const float* v = nullptr;
  size_t n = 0;
  float thr = 0.f, var = 0.f;
  ev_row(r, y, nb, &v, &n, &thr, &var);  // a row with runs exists
  const size_t base = (size_t)t * EV_TILE;
#pragma unroll
  for (int i = 0; i < EV_PER; i++) {
    const size_t li = (size_t)i * EV_THREADS + tid, j = base + li;
    sv[li] = j < n ? v[j] : NAN;
  }
  if (tid == 0) s_before = base > 0 && v[base - 1] > thr;
  __syncthreads();
  // this thread's samples [c0, c0 + EV_PER): its run starts and its leading fragment
  const int c0 = tid * EV_PER;
  unsigned starts = 0, plen = 0, parg = 0;
  float pmax = 0.f;
  bool lead = true, prev = tid == 0 ? s_before : sv[c0 - 1] > thr;
  for (int e = 0; e < EV_PER; e++) {
    const float x = sv[c0 + e];
    const bool a = x > thr;
    starts += (a && !prev) ? 1u : 0u;
    if (lead && a) {
      if (plen == 0 || x > pmax) {
        pmax = x;
        parg = (unsigned)e;
      }
      plen++;
    } else {
      lead = false;
    }
    prev = a;
  }
  s_plen[tid] = plen;
  s_pmax[tid] = pmax;
  s_parg[tid] = parg;
  // exclusive scan of the threads' run counts: each run's rank within the tile
  unsigned incl = starts;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  if (lane == 31) s_w[wid] = incl;
  __syncthreads();
  unsigned rank = incl - starts;
  for (int w = 0; w < wid; w++) rank += s_w[w];
  if (starts == 0) return;
  unsigned long long slot = offset[row0 + t] + rank;
  prev = tid == 0 ? s_before : sv[c0 - 1] > thr;
  for (int e = 0; e < EV_PER; e++) {
    const bool a = sv[c0 + e] > thr;
    const bool is_start = a && !prev;
    prev = a;
    if (!is_start) continue;
    const size_t begin = base + c0 + e;
    float m = sv[c0 + e];
    size_t arg = begin, end = 0;
    int q = e + 1;
    for (; q < EV_PER; q++) {
      const float x = sv[c0 + q];
      if (!(x > thr)) break;
      if (x > m) {
        m = x;
        arg = base + c0 + q;
      }
    }
    if (q < EV_PER) {
      end = base + c0 + q;
    } else {
      bool done = false;
      for (int u = tid + 1; u < EV_THREADS && !done; u++) {  // the following threads' fragments
        const unsigned pl = s_plen[u];
        if (pl > 0 && s_pmax[u] > m) {
          m = s_pmax[u];
          arg = base + (size_t)u * EV_PER + s_parg[u];
        }
        if (pl < EV_PER) {
          end = base + (size_t)u * EV_PER + pl;
          done = true;
        }
      }
      for (size_t tt = (size_t)t + 1; !done; tt++) {  // the following tiles' summaries
        const size_t b2 = tt * EV_TILE;
        if (b2 >= n) {
          end = n;
          break;
        }
        const ev_tile f = tile[row0 + tt];
        if (f.prefix_len > 0 && f.prefix_max > m) {
          m = f.prefix_max;
          arg = b2 + f.prefix_arg;
        }
        if ((size_t)f.prefix_len < min((size_t)EV_TILE, n - b2)) {
          end = b2 + f.prefix_len;
          done = true;
        }
      }
    }
    if (slot < max_events)
      out[slot] = ev_event{begin, end, arg, var > 0.f ? m / sqrtf(var) : 0.f, r.trial0 + y, nb, r.stream};
    slot++;
  }
}

}  // namespace srtb_b200
