// srtb_b200.cu — C-ABI implementation (include/srtb_b200.h): context, FFT planning,
// kernel launches. Host logic only mirrors the reference's host-side arithmetic; every
// data-path byte is touched by the CUDA kernels in fft_engine.cuh / ops_kernels.cuh.
// There is no CPU fallback.
#include <cuda.h>  // CUtensorMap types only; the encoder is fetched with cudaGetDriverEntryPoint
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <optional>
#include <set>
#include <string>
#include <vector>

#include "../../include/srtb_b200.h"
#include "fft_engine.cuh"
#include "fft_bigrow.cuh"
#include "ops_kernels.cuh"
#include "thumbnail.cuh"
#include "correlator.cuh"
#include "incoherent.cuh"
#include "stream_sum.cuh"
#include "fold.cuh"
#include "events.cuh"
#include "cutout.cuh"

using namespace srtb_b200;

static thread_local std::string g_last_error;

// result headers per block: one per data stream (at most 4), then the total-intensity sum's (signal_detect_sum_streams)
constexpr int RES_GROUP = 5, SUM_SLOT = 4;
// the device's records are the ABI's structs, copied byte for byte
static_assert(sizeof(detect_dev_result) == sizeof(srtb_b200_detect_result), "result layout");
static_assert(sizeof(detect_dev_peak) == sizeof(srtb_b200_peak), "peak layout");
static_assert(sizeof(ev_event) == sizeof(srtb_b200_event) && sizeof(ev_event) == 40, "event layout");
// head of a lane's event scratch and of a pinned event list: the counts [RES_GROUP] (and the scratch's ticket)
constexpr size_t EV_HEAD = 256;

// an allocation the context owns, device memory or (PINNED) pinned host memory, freed with its owner. grow() sizes it;
// move-only, so a lane_state holding some stays swappable (lane_swap)
template <class T, bool PINNED = false>
struct buffer {
  T* p = nullptr;
  size_t bytes = 0;
  buffer() = default;
  buffer(buffer&& o) noexcept : p(o.p), bytes(o.bytes) {
    o.p = nullptr;
    o.bytes = 0;
  }
  buffer& operator=(buffer&& o) noexcept {
    std::swap(p, o.p);
    std::swap(bytes, o.bytes);
    return *this;
  }
  ~buffer() { release(); }
  cudaError_t release() {
    const cudaError_t e = !p ? cudaSuccess : PINNED ? cudaFreeHost(p) : cudaFree(p);
    p = nullptr;
    bytes = 0;
    return e;
  }
};

// what one chain of kernels writes through: the data streams of a block are independent until their result headers
// are read back, so a context runs the odd-numbered ones on a second lane with its own CUDA stream and scratch (one
// lane's kernel tails and small detector kernels overlap the other lane's FFT sweeps)
struct lane_state {
  cudaStream_t stream = nullptr;
  buffer<float2> fft_scratch;
  // s1
  double* partial = nullptr;
  unsigned* ticket = nullptr;
  unsigned* detect_ticket = nullptr;  // last-CTA ticket of the detector's column-sum kernel
  float* mean = nullptr;
  // detect
  buffer<float> colsum_partial, acc;
  // long waterfall rows: per-tile SK statistics of the last sweep, per-row zap flags
  buffer<float2> long_stats;
  buffer<unsigned char> long_zap;
  // events (events.cuh): the running event counts [RES_GROUP] and the count kernel's ticket at the head (EV_HEAD
  // bytes), then the tile summaries, scan offsets and uploaded headers of one pass (ev_scratch_for)
  buffer<char> ev_work;
};

// a pinned event list: the counts [RES_GROUP] in an EV_HEAD-byte head, then [rows][max_events] events the emit kernel
// writes through
struct ev_list {
  char* p = nullptr;
  size_t max_events = 0;
  unsigned long long* counts() const { return reinterpret_cast<unsigned long long*>(p); }
  ev_event* row(size_t r) const { return reinterpret_cast<ev_event*>(p + EV_HEAD) + r * max_events; }
};

// one block in flight on the pipelined ingest ring (submit_ring / collect_ring)
struct ring_slot {
  buffer<void> baseband;  // the block's host baseband, copied on the copy stream
  cudaEvent_t h2d = nullptr, done = nullptr, done_alt = nullptr;  // done_alt: the second lane's completion of the block
  int streams = 0, ticket = 0;
  bool busy = false, alt_used = false, sum = false;  // sum: the block carries the total-intensity sum's header
  // outputs: ctx-owned working buffers / pinned series unless the caller supplied its own (submit_block_ex)
  buffer<float> stream_buf[4];
  buffer<float, true> h_series;
  float* out_spectrum[4] = {};
  float* out_series = nullptr;
  // events (submit_block_events): the pinned list [streams (+1)][max_events], kept and grown like h_series; list is
  // into it, or {null, 0} when the block lists no events
  buffer<char, true> ev;
  ev_list list;
};

// what the incoherent search needs of (C, band, dm, trials): incoherent_plan_for
struct incoherent_plan {
  std::vector<int64_t> shifts;       // [n_dm][C]
  uint64_t s_plus = 0, s_minus = 0;
  std::vector<int> order;            // [n_dm] trial at each sorted position
  std::vector<int2> groups, gspan;   // [groups] (first, count); [groups][C] (min, max) of a group's s + S-
  unsigned spread = 0;               // largest max - min of any group and channel
};

struct srtb_b200_ctx {
  // a context may be shared by the threads of a pipeline (the reference hands one sycl::queue to every pipe): every
  // C-ABI entry takes this lock, so the planning state below (tables, scratch sizes, kernel attributes) is never
  // mutated concurrently. Recursive because the block entries call the stage entries.
  std::recursive_mutex mu;
  int device = 0;
  int sm_count = 132;
  std::string err;
  uint64_t launches = 0;
  std::set<const void*> configured;  // kernels whose smem attribute is set on this device
  std::map<const void*, int> occupancy;  // resident CTAs per SM of the persistent kernels
  // the lane the launch code writes through, and the other one. lane_swap() exchanges them, so the launch code itself
  // is lane-agnostic. The first lane's stream is the caller's; the second lane (created on first use) owns its stream.
  lane_state lane, alt;
  bool alt_ready = false, on_alt = false;
  int lanes = 1;  // SRTB_B200_LANES (default 2): CUDA streams per context the data streams of a block are spread over
  cudaEvent_t lane_fork = nullptr, lane_join = nullptr;
  // FFT
  buffer<float2> tw[13];
  std::map<int, buffer<float2>> bigtw;  // log2(n_i) -> [3 << q]
  buffer<float2> bigrow_tab[2][2];      // [logl - 13][forward] whole-row kernel tables
  // detect (slots = streams in flight, then SUM_SLOT)
  buffer<float> series[RES_GROUP];
  detect_dev_result* d_res = nullptr;  // RES_GROUP slots
  detect_dev_result* h_res = nullptr;  // pinned, RES_GROUP slots for process_block, then RES_GROUP per ring slot
  size_t series_len[RES_GROUP] = {};  // time_count of the slot's last detector run: the row stride of its series
  // total-intensity sum: the streams' raw column sums [1 + RING_SLOTS][4][L] (group 0: process_block, 1 + slot: the
  // ring; slot-owned, so a lane's next block cannot overwrite what the sum of this one still reads), and the mask
  // kernel's output (mask float2[C], mismatched channels uint2[C], their count)
  buffer<float> sum_raw;
  buffer<float2> sum_mask;
  // pipelined ingest ring
  cudaStream_t copy_stream = nullptr;
  ring_slot ring[SRTB_B200_RING_SLOTS];
  uint64_t submit_count = 0;
  // DM sweep working copy of the spectrum, per-trial result headers
  buffer<float2> sweep_buf;
  buffer<detect_dev_result> sweep_res;
  // optional per-stage timing (srtb_b200_stage_stats)
  bool stats_on = false;
  cudaEvent_t stat_ev[SRTB_B200_STAGE_COUNT][2] = {};
  double stat_bytes[SRTB_B200_STAGE_COUNT] = {};
  bool stat_have[SRTB_B200_STAGE_COUNT] = {};
  bool pdl_auto = false;  // programmatic dependent launch for the current block (short kernels only)
  // process_block
  buffer<void> d_baseband;
  buffer<float> stream_buf[4];
  // K12 phase table of the current (block geometry, DM): see chirp_phase_table_kernel
  buffer<float> chirp_tab;
  double chirp_tab_key[6] = {0, 0, 0, 0, 0, 0};  // n, f_min, df, inv_fc, f_c, ddm
  // simplify_spectrum: row-resampled intensities R[C][W] and the column stage's per-CTA partial sums
  buffer<float> thumb_rows, thumb_partial;
  // correlate: the two inputs' in-place R2C buffers of real_count + 2 floats
  buffer<float> corr_buf[2];
  // correlate_accumulate / _finish: the packed segment rows of both inputs (also finish's Ms-point C2C buffer), the
  // split's per-row-group partial sums and its per-bin-tile tickets (sm_count * 8, zero between launches)
  buffer<float2> corr_rows;
  buffer<double2> corr_partial;
  unsigned* corr_tickets = nullptr;
  // incoherent DM search: the plan of the last (geometry, dm, trial list) and its key, the kernel's offsets [C][n_dm]
  // (s + S- in sorted order) and whether inc_tab holds them; the device tables, and the per-trial series
  // [n_dm][nb][T], scans [n_dm][T], result headers, peaks and tickets
  struct {
    std::vector<double> key;
    incoherent_plan plan;
    std::vector<int> off;
    bool uploaded = false;
  } inc;
  buffer<char> inc_tab, inc_work;
  // fold: the sorted bin plan, hits, profile and kept, and the per-CTA rows fold_finish_kernel adds (srtb_b200_fold)
  buffer<char> fold_work;
  // the DM searches' and series_events' event list (their scratch is the first lane's)
  buffer<char, true> ev_host;
  // candidate_cutouts: the tables, decimated power rows and images of one call (cutout_layout)
  buffer<char> cut_work;
};

static void lane_swap(srtb_b200_ctx* ctx) {
  std::swap(ctx->lane, ctx->alt);
  ctx->on_alt = !ctx->on_alt;
}

// the fixed-size device state of a lane (its stream is set by the caller)
static cudaError_t lane_alloc(lane_state* l) {
  cudaError_t e = cudaMalloc(&l->partial, sizeof(double) * 4096);
  if (e == cudaSuccess) e = cudaMalloc(&l->ticket, sizeof(unsigned));
  if (e == cudaSuccess) e = cudaMemset(l->ticket, 0, sizeof(unsigned));
  if (e == cudaSuccess) e = cudaMalloc(&l->detect_ticket, sizeof(unsigned));
  if (e == cudaSuccess) e = cudaMemset(l->detect_ticket, 0, sizeof(unsigned));
  if (e == cudaSuccess) e = cudaMalloc(&l->mean, sizeof(float));
  return e;
}

#define API_LOCK(c)                                         \
  std::unique_lock<std::recursive_mutex> api_lock_;         \
  if (c) api_lock_ = std::unique_lock<std::recursive_mutex>((c)->mu)

static int fail(srtb_b200_ctx* ctx, int code, const std::string& msg) {
  g_last_error = msg;
  if (ctx) ctx->err = msg;
  return code;
}

#define CK(call)                                                                          \
  do {                                                                                    \
    cudaError_t e_ = (call);                                                              \
    if (e_ != cudaSuccess)                                                                \
      return fail(ctx, SRTB_B200_E_CUDA,                                                  \
                  std::string(#call) + ": " + cudaGetErrorString(e_) + " (" __FILE__ ":" + \
                      std::to_string(__LINE__) + ")");                                    \
  } while (0)

// both lanes of the context idle (before anything either of them may still use is freed)
static int sync_lanes(srtb_b200_ctx* ctx) {
  CK(cudaStreamSynchronize(ctx->lane.stream));
  if (ctx->alt_ready) CK(cudaStreamSynchronize(ctx->alt.stream));
  return 0;
}

// b holds at least `bytes` afterwards: a larger allocation replaces a smaller one once both lanes are idle. A failed
// allocation leaves b empty and clears the runtime's last error, which the next launch check would otherwise report.
template <class T, bool PINNED>
static int grow(srtb_b200_ctx* ctx, buffer<T, PINNED>& b, size_t bytes) {
  if (b.bytes >= bytes && b.p) return 0;
  if (b.p) {
    if (int rc = sync_lanes(ctx)) return rc;
    CK(b.release());
  }
  void* q = nullptr;
  const cudaError_t e = PINNED ? cudaMallocHost(&q, bytes) : cudaMalloc(&q, bytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(ctx, SRTB_B200_E_NOMEM, std::string(PINNED ? "cudaMallocHost(" : "cudaMalloc(") + std::to_string(bytes) +
                                            "): " + cudaGetErrorString(e));
  }
  b.p = static_cast<T*>(q);
  b.bytes = bytes;
  return 0;
}

static inline bool is_pow2(size_t n) { return n && !(n & (n - 1)); }
static inline bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7u) == 0; }
static inline int ilog2(size_t n) {
  int k = 0;
  while (((size_t)1 << k) < n) k++;
  return k;
}
static inline unsigned grid_for(const srtb_b200_ctx* ctx, size_t work_items, int threads, int per_sm = 8) {
  const size_t need = (work_items + threads - 1) / threads;
  const size_t cap = (size_t)ctx->sm_count * per_sm;
  return (unsigned)std::max<size_t>(1, std::min(need, cap));
}

// Every counted kernel launch goes through here, so srtb_b200_launch_count counts each launch the runtime accepted.
// Returns the launch's error, else cudaGetLastError().
template <typename... KArgs, typename... Args>
static cudaError_t launch(srtb_b200_ctx* ctx, const cudaLaunchConfig_t& cfg, void (*kern)(KArgs...), Args&&... args) {
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
  if (e != cudaSuccess) return e;
  ctx->launches++;
  return cudaGetLastError();
}

// A launch on the current lane's stream. pdl: programmatic dependent launch along the block path (ctx->pdl_auto): the
// kernel's set-up (tables into shared memory, barriers) overlaps its predecessor's tail, so such a kernel must call
// pdl_wait() before touching anything a predecessor produces. It pays where kernels are short (2^24-sample blocks) and
// can cost where they are long, since the early-resident CTAs of the next kernel only take shared memory from the
// running one. Hence: on for blocks up to 2^25 samples, off above and outside a block.
template <typename... KArgs, typename... Args>
static cudaError_t launch(srtb_b200_ctx* ctx, bool pdl, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem,
                          Args&&... args) {
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr.val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = ctx->lane.stream;
  cfg.attrs = &attr;
  cfg.numAttrs = pdl && ctx->pdl_auto ? 1 : 0;
  return launch(ctx, cfg, kern, std::forward<Args>(args)...);
}

// a kernel's dynamic shared-memory limit, set once per context to `bytes`: the largest size any of its launches asks for
template <class K>
static int set_smem_max(srtb_b200_ctx* ctx, K kern, size_t bytes) {
  const void* key = reinterpret_cast<const void*>(kern);
  if (ctx->configured.count(key)) return 0;
  CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  ctx->configured.insert(key);
  return 0;
}

// grid of a persistent kernel: ntiles CTAs, at most one wave (resident CTAs per SM found once, at the smem of the first
// launch, under a limit of smem_max)
template <class K>
static int persistent_grid(srtb_b200_ctx* ctx, K kern, int threads, size_t smem, size_t smem_max, size_t ntiles,
                           unsigned* grid) {
  if (int rc = set_smem_max(ctx, kern, smem_max)) return rc;
  const void* key = reinterpret_cast<const void*>(kern);
  if (!ctx->occupancy.count(key)) {
    int per_sm = 1;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem));
    ctx->occupancy[key] = std::max(1, per_sm);
  }
  *grid = (unsigned)std::min<size_t>(ntiles, (size_t)ctx->sm_count * ctx->occupancy[key]);
  return 0;
}

// records a CUDA-event pair around one stage call when per-stage statistics are enabled
struct stage_scope {
  srtb_b200_ctx* ctx;
  int stage;
  stage_scope(srtb_b200_ctx* c, int st, double bytes) : ctx(c), stage(st) {
    if (!ctx->stats_on) {
      ctx = nullptr;
      return;
    }
    if (!ctx->stat_ev[stage][0]) {
      cudaEventCreate(&ctx->stat_ev[stage][0]);
      cudaEventCreate(&ctx->stat_ev[stage][1]);
    }
    ctx->stat_bytes[stage] = bytes;
    ctx->stat_have[stage] = true;
    cudaEventRecord(ctx->stat_ev[stage][0], ctx->lane.stream);
  }
  ~stage_scope() {
    if (ctx) cudaEventRecord(ctx->stat_ev[stage][1], ctx->lane.stream);
  }
};

extern "C" {

const char* srtb_b200_version(void) { return "srtb_b200 0.1 (sm_90a)"; }

int srtb_b200_ctx_create(int device, void* cuda_stream, srtb_b200_ctx** out) {
  srtb_b200_ctx* ctx = nullptr;
  if (!out) return fail(nullptr, SRTB_B200_E_INVALID, "ctx_create: out is null");
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0)
    return fail(nullptr, SRTB_B200_E_CUDA,
                std::string("ctx_create: no CUDA device (") + cudaGetErrorString(e) +
                    "); libsrtb_b200 has no CPU fallback");
  if (device < 0 || device >= count) return fail(nullptr, SRTB_B200_E_INVALID, "ctx_create: bad device index");
  ctx = new srtb_b200_ctx();
  ctx->device = device;
  ctx->lane.stream = static_cast<cudaStream_t>(cuda_stream);
  e = cudaSetDevice(device);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device);
  if (e == cudaSuccess) e = lane_alloc(&ctx->lane);
  if (e == cudaSuccess) e = cudaMalloc(&ctx->d_res, sizeof(detect_dev_result) * RES_GROUP);
  if (e == cudaSuccess) e = cudaMemset(ctx->d_res, 0, sizeof(detect_dev_result) * RES_GROUP);
  if (e == cudaSuccess) e = cudaMallocHost(&ctx->h_res, sizeof(detect_dev_result) * RES_GROUP * (1 + SRTB_B200_RING_SLOTS));
  if (e != cudaSuccess) {
    const std::string msg = std::string("ctx_create: ") + cudaGetErrorString(e);
    srtb_b200_ctx_destroy(ctx);  // frees whatever was allocated before the failure
    return fail(nullptr, SRTB_B200_E_CUDA, msg);
  }
  if (const char* v = std::getenv("SRTB_B200_LANES")) ctx->lanes = std::atoi(v) >= 2 ? 2 : 1;
  else ctx->lanes = 2;
  *out = ctx;
  return 0;
}

int srtb_b200_ctx_destroy(srtb_b200_ctx* ctx) {
  if (!ctx) return 0;
  cudaSetDevice(ctx->device);
  if (ctx->on_alt) lane_swap(ctx);
  cudaStreamSynchronize(ctx->lane.stream);
  if (ctx->alt_ready) {
    cudaStreamSynchronize(ctx->alt.stream);
    cudaStreamDestroy(ctx->alt.stream);
  }
  for (lane_state* l : {&ctx->lane, &ctx->alt}) {
    cudaFree(l->partial);
    cudaFree(l->ticket);
    cudaFree(l->detect_ticket);
    cudaFree(l->mean);
  }
  cudaFree(ctx->d_res);
  cudaFreeHost(ctx->h_res);
  cudaFree(ctx->corr_tickets);
  if (ctx->lane_fork) cudaEventDestroy(ctx->lane_fork);
  if (ctx->lane_join) cudaEventDestroy(ctx->lane_join);
  for (ring_slot& rs : ctx->ring) {
    if (rs.h2d) cudaEventDestroy(rs.h2d);
    if (rs.done) cudaEventDestroy(rs.done);
    if (rs.done_alt) cudaEventDestroy(rs.done_alt);
  }
  if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
  for (auto& ev : ctx->stat_ev)
    for (auto& e2 : ev)
      if (e2) cudaEventDestroy(e2);
  delete ctx;  // the buffers free themselves
  return 0;
}

int srtb_b200_ctx_set_stream(srtb_b200_ctx* ctx, void* cuda_stream) {
  API_LOCK(ctx);
  if (!ctx) return fail(nullptr, SRTB_B200_E_INVALID, "set_stream: ctx is null");
  ctx->lane.stream = static_cast<cudaStream_t>(cuda_stream);
  return 0;
}

int srtb_b200_synchronize(srtb_b200_ctx* ctx) {
  if (!ctx) return fail(nullptr, SRTB_B200_E_INVALID, "synchronize: ctx is null");
  cudaStream_t s0, s1 = nullptr;
  {
    API_LOCK(ctx);  // the wait itself runs unlocked: other threads keep enqueueing meanwhile
    s0 = ctx->on_alt ? ctx->alt.stream : ctx->lane.stream;
    if (ctx->alt_ready) s1 = ctx->on_alt ? ctx->lane.stream : ctx->alt.stream;
  }
  CK(cudaStreamSynchronize(s0));
  if (s1) CK(cudaStreamSynchronize(s1));
  return 0;
}

const char* srtb_b200_last_error(const srtb_b200_ctx* ctx) {
  return ctx ? ctx->err.c_str() : g_last_error.c_str();
}

uint64_t srtb_b200_launch_count(const srtb_b200_ctx* ctx) { return ctx ? ctx->launches : 0; }

int srtb_b200_stage_stats_enable(srtb_b200_ctx* ctx, int on) {
  API_LOCK(ctx);
  if (!ctx) return fail(nullptr, SRTB_B200_E_INVALID, "stage_stats_enable: ctx is null");
  ctx->stats_on = on != 0;
  return 0;
}

int srtb_b200_stage_stats(srtb_b200_ctx* ctx, int stage, double* ms, double* bytes) {
  API_LOCK(ctx);
  if (!ctx || !ms || !bytes) return fail(ctx, SRTB_B200_E_INVALID, "stage_stats: null argument");
  if (stage < 0 || stage >= SRTB_B200_STAGE_COUNT) return fail(ctx, SRTB_B200_E_INVALID, "stage_stats: unknown stage");
  if (!ctx->stat_have[stage]) return fail(ctx, SRTB_B200_E_INVALID, "stage_stats: stage not timed yet (enable first)");
  CK(cudaSetDevice(ctx->device));
  CK(cudaEventSynchronize(ctx->stat_ev[stage][1]));
  float t = 0.f;
  CK(cudaEventElapsedTime(&t, ctx->stat_ev[stage][0], ctx->stat_ev[stage][1]));
  *ms = t;
  *bytes = ctx->stat_bytes[stage];
  return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------
// unpack
// ------------------------------------------------------------------------------------
template <int BITS>
static int launch_unpack_simple(srtb_b200_ctx* ctx, const void* d_in, float* out, size_t n, int window) {
  const bool aligned = ((reinterpret_cast<uintptr_t>(d_in) & 15u) == 0) &&
                       ((reinterpret_cast<uintptr_t>(out) & 15u) == 0);
  if (!aligned) {
    CK(launch(ctx, false, unpack_simple_scalar_kernel<BITS>, grid_for(ctx, n, 256), 256, 0, d_in, out, n, window));
  } else {
    auto kern = window == 0 ? unpack_simple_kernel<BITS, false> : unpack_simple_kernel<BITS, true>;
    CK(launch(ctx, false, kern, grid_for(ctx, n / 16 + 1, 256), 256, 0, d_in, out, n, window));
  }
  return 0;
}

template <int BITS>
static int launch_unpack_il2(srtb_b200_ctx* ctx, const void* d_in, float* o1, float* o2, size_t n, int window) {
  CK(launch(ctx, false, unpack_interleaved2_kernel<BITS>, grid_for(ctx, n / 4 + 1, 256), 256, 0, d_in, o1, o2, n, window));
  return 0;
}

extern "C" int srtb_b200_unpack(srtb_b200_ctx* ctx, const void* d_in, size_t in_bytes, int bits,
                                int format, int window, float* const d_out[4], size_t out_count) {
  API_LOCK(ctx);
  if (!ctx || !d_in || !d_out || !d_out[0]) return fail(ctx, SRTB_B200_E_INVALID, "unpack: null argument");
  if (window < 0 || window > 2) return fail(ctx, SRTB_B200_E_INVALID, "unpack: unknown window");
  if (out_count == 0) return 0;
  const int abits = bits < 0 ? -bits : bits;
  stage_scope stats_(ctx, SRTB_B200_STAGE_UNPACK, (double)in_bytes + 4.0 * (double)out_count * (format == SRTB_B200_FORMAT_SIMPLE ? 1 : (format == SRTB_B200_FORMAT_GZNUPSR_A1_4 ? 4 : 2)));
  int streams = 1;
  if (format == SRTB_B200_FORMAT_INTERLEAVED_2 || format == SRTB_B200_FORMAT_NAOCPSR_SNAP1 ||
      format == SRTB_B200_FORMAT_GZNUPSR_A1_2)
    streams = 2;
  else if (format == SRTB_B200_FORMAT_GZNUPSR_A1_4)
    streams = 4;
  else if (format != SRTB_B200_FORMAT_SIMPLE)
    return fail(ctx, SRTB_B200_E_UNSUPPORTED, "[start_unpack_pipe] Unknown format name: " + std::to_string(format));
  if (abits == 0 || (size_t)out_count * streams * abits > in_bytes * 8)
    return fail(ctx, SRTB_B200_E_INVALID, "unpack: in_bytes too small for out_count");
  for (int s = 0; s < streams; s++)
    if (!d_out[s]) return fail(ctx, SRTB_B200_E_INVALID, "unpack: null output stream");
  if (streams == 1) {
    // the scalar fall-back loads one sample at a time: 16/32/64-bit samples need their natural alignment
    const uintptr_t width = abits >= 16 ? (uintptr_t)(abits / 8) : 1u;
    if (reinterpret_cast<uintptr_t>(d_in) % width)
      return fail(ctx, SRTB_B200_E_INVALID, "unpack: d_in is not aligned to the " + std::to_string(width) + "-byte sample width");
    if (reinterpret_cast<uintptr_t>(d_out[0]) & 3u) return fail(ctx, SRTB_B200_E_INVALID, "unpack: d_out[0] is not 4-byte aligned");
  }
  if (streams > 1) {
    // the multi-stream kernels move 8/16-byte words: the board formats are int8 only, whole 4-sample words, and
    // every buffer 16-byte aligned (the single-stream path has a scalar fall-back, these do not)
    if ((format == SRTB_B200_FORMAT_GZNUPSR_A1_2 || format == SRTB_B200_FORMAT_GZNUPSR_A1_4) && abits != 8)
      return fail(ctx, SRTB_B200_E_UNSUPPORTED, "gznupsr_a1 requires 8-bit samples, got baseband_input_bits = " + std::to_string(bits));
    if ((format == SRTB_B200_FORMAT_GZNUPSR_A1_2 || format == SRTB_B200_FORMAT_GZNUPSR_A1_4) && (out_count & 3))
      return fail(ctx, SRTB_B200_E_SIZE, "gznupsr_a1: samples per stream must be a multiple of 4, got " + std::to_string(out_count));
    bool aligned = (reinterpret_cast<uintptr_t>(d_in) & 15u) == 0;
    for (int s = 0; s < streams; s++) aligned = aligned && (reinterpret_cast<uintptr_t>(d_out[s]) & 15u) == 0;
    if (!aligned) return fail(ctx, SRTB_B200_E_INVALID, "unpack: multi-stream formats need 16-byte aligned input and output buffers");
  }
  CK(cudaSetDevice(ctx->device));
  switch (format) {
    case SRTB_B200_FORMAT_SIMPLE:
      switch (bits) {
        case 1: return launch_unpack_simple<1>(ctx, d_in, d_out[0], out_count, window);
        case 2: return launch_unpack_simple<2>(ctx, d_in, d_out[0], out_count, window);
        case 4: return launch_unpack_simple<4>(ctx, d_in, d_out[0], out_count, window);
        case 8: return launch_unpack_simple<8>(ctx, d_in, d_out[0], out_count, window);
        case -8: return launch_unpack_simple<-8>(ctx, d_in, d_out[0], out_count, window);
        case 16: return launch_unpack_simple<16>(ctx, d_in, d_out[0], out_count, window);
        case -16: return launch_unpack_simple<-16>(ctx, d_in, d_out[0], out_count, window);
        case 32: return launch_unpack_simple<32>(ctx, d_in, d_out[0], out_count, window);
        case 64: return launch_unpack_simple<64>(ctx, d_in, d_out[0], out_count, window);
        default:
          return fail(ctx, SRTB_B200_E_UNSUPPORTED,
                      "[unpack pipe] unsupported baseband_input_bits = " + std::to_string(bits));
      }
    case SRTB_B200_FORMAT_INTERLEAVED_2:
      switch (bits) {
        case 8: return launch_unpack_il2<8>(ctx, d_in, d_out[0], d_out[1], out_count, window);
        case -8: return launch_unpack_il2<-8>(ctx, d_in, d_out[0], d_out[1], out_count, window);
        case 16: return launch_unpack_il2<16>(ctx, d_in, d_out[0], d_out[1], out_count, window);
        case -16: return launch_unpack_il2<-16>(ctx, d_in, d_out[0], d_out[1], out_count, window);
        case 32: return launch_unpack_il2<32>(ctx, d_in, d_out[0], d_out[1], out_count, window);
        case 64: return launch_unpack_il2<64>(ctx, d_in, d_out[0], d_out[1], out_count, window);
        default:
          return fail(ctx, SRTB_B200_E_UNSUPPORTED,
                      "[unpack_2pol_interleave_pipe] unsupported baseband_input_bits = " + std::to_string(bits));
      }
    case SRTB_B200_FORMAT_NAOCPSR_SNAP1:
      if (bits != -8)
        return fail(ctx, SRTB_B200_E_UNSUPPORTED, "naocpsr_snap1 requires baseband_input_bits = -8");
      CK(launch(ctx, false, unpack_snap1_kernel, grid_for(ctx, out_count / 4 + 1, 256), 256, 0, d_in, d_out[0], d_out[1],
                out_count, window));
      break;
    case SRTB_B200_FORMAT_GZNUPSR_A1_2:
      CK(launch(ctx, false, unpack_gznupsr_kernel<2>, grid_for(ctx, out_count / 4 + 1, 256), 256, 0, d_in, d_out[0],
                d_out[1], nullptr, nullptr, out_count, window));
      break;
    case SRTB_B200_FORMAT_GZNUPSR_A1_4:
      CK(launch(ctx, false, unpack_gznupsr_kernel<4>, grid_for(ctx, out_count / 4 + 1, 256), 256, 0, d_in, d_out[0],
                d_out[1], d_out[2], d_out[3], out_count, window));
      break;
  }
  return 0;
}

// ------------------------------------------------------------------------------------
// FFT planning + launches
// ------------------------------------------------------------------------------------
// a constant table on the device, uploaded synchronously so that both lanes and every later launch may read it; d is
// set only once the upload has completed
static int upload_table(srtb_b200_ctx* ctx, const std::vector<float2>& h, buffer<float2>* d) {
  buffer<float2> t;
  void* q = nullptr;
  CK(cudaMalloc(&q, h.size() * sizeof(float2)));
  t.p = static_cast<float2*>(q);
  t.bytes = h.size() * sizeof(float2);
  CK(cudaMemcpyAsync(t.p, h.data(), t.bytes, cudaMemcpyHostToDevice, ctx->lane.stream));
  CK(cudaStreamSynchronize(ctx->lane.stream));
  *d = std::move(t);
  return 0;
}

static int get_stage_twiddles(srtb_b200_ctx* ctx, int logl, const float2** out) {
  if (!ctx->tw[logl].p) {
    const size_t L = (size_t)1 << logl;
    std::vector<float2> h(L);
    for (size_t j = 0; j < L; j++) {
      const double a = -2.0 * M_PI * (double)j / (double)L;
      h[j] = make_float2((float)std::cos(a), (float)std::sin(a));
    }
    if (int rc = upload_table(ctx, h, &ctx->tw[logl])) return rc;
  }
  *out = ctx->tw[logl].p;
  return 0;
}

static int get_big_twiddles(srtb_b200_ctx* ctx, int logn, big_twiddle* out) {
  const int q = (logn + 2) / 3;
  buffer<float2>& d = ctx->bigtw[logn];
  if (!d.p) {
    const size_t n = (size_t)1 << logn, m = (size_t)1 << q;
    std::vector<float2> h(3 * m);
    for (int level = 0; level < 3; level++)
      for (size_t j = 0; j < m; j++) {
        const size_t idx = (j << (level * q)) & (n - 1);
        const double a = -2.0 * M_PI * (double)idx / (double)n;
        h[level * m + j] = make_float2((float)std::cos(a), (float)std::sin(a));
      }
    if (int rc = upload_table(ctx, h, &d)) return rc;
  }
  out->tab = d.p;
  out->q = q;
  return 0;
}

template <int LOGL, int T, int MODE, bool FWD, class IO>
static int launch_pass(srtb_b200_ctx* ctx, const IO& io, unsigned grid, size_t extra_smem) {
  auto kern = fft_pass_kernel<LOGL, T, MODE, FWD, IO>;
  const size_t smem = (size_t)tile_layout<LOGL, T, MODE>::ELEMS * sizeof(float2) + extra_smem;
  if (smem > 48 * 1024)
    if (int rc = set_smem_max(ctx, kern, 200 * 1024)) return rc;
  const float2* tw = nullptr;
  if (int rc = get_stage_twiddles(ctx, LOGL, &tw)) return rc;
  CK(launch(ctx, false, kern, grid, pass_threads<LOGL, T>::value, smem, io, tw));
  return 0;
}

// rows per CTA in ROW mode: 256 threads up to L = 2048, 512 threads for L = 4096
template <int LOGL>
struct row_t {
  static constexpr int value = (LOGL >= 11) ? 1 : (1 << (11 - LOGL));
};
template <int LOGL>
struct col_t {
  static constexpr int value = (LOGL <= 8) ? 16 : 8;
};

// sixteen-points-per-thread row kernels (L = 256 .. 4096); shorter rows take the eight-point kernel
template <int LOGL>
struct has_row16 {
  static constexpr bool value = (LOGL >= 8 && LOGL <= 12);
};

template <int LOGL, bool FWD>
static int launch_row(srtb_b200_ctx* ctx, const float2* in, float2* out, size_t nrows) {
  constexpr int T = row_t<LOGL>::value;
  if constexpr (has_row16<LOGL>::value) {
    if ((reinterpret_cast<uintptr_t>(in) & 15u) == 0) {
      constexpr int T16 = row16_t<LOGL>::value, threads = ((1 << LOGL) / 16) * T16;
      auto kern = fft_row16_tma_kernel<LOGL, T16, FWD>;
      constexpr size_t smem = row16_smem<LOGL, T16>::bytes;
      const size_t ntiles = (nrows + T16 - 1) / T16;
      unsigned grid = 1;
      if (int rc = persistent_grid(ctx, kern, threads, smem, smem, ntiles, &grid)) return rc;
      const float2* tw = nullptr;
      if (int rc = get_stage_twiddles(ctx, LOGL, &tw)) return rc;
      CK(launch(ctx, true, kern, grid, threads, smem, in, out, nrows, tw, row_sk_params{}, row_chirp_params{}));
      return 0;
    }
  } else if ((reinterpret_cast<uintptr_t>(in) & 15u) == 0) {
    // persistent TMA-fed kernel (cp.async.bulk needs 16-byte aligned rows)
    auto kern = fft_row_tma_kernel<LOGL, T, FWD>;
    constexpr int threads = pass_threads<LOGL, T>::value;
    constexpr size_t smem = row_tma_smem<LOGL, T>::bytes;
    unsigned grid = 1;
    if (int rc = persistent_grid(ctx, kern, threads, smem, smem, (nrows + T - 1) / T, &grid)) return rc;
    const float2* tw = nullptr;
    if (int rc = get_stage_twiddles(ctx, LOGL, &tw)) return rc;
    CK(launch(ctx, false, kern, grid, threads, smem, in, out, nrows, tw, row_sk_params{}));
    return 0;
  }
  row_io<LOGL, T> io;
  io.in = in;
  io.out = out;
  io.nrows = nrows;
  io.row0 = 0;
  const unsigned grid = (unsigned)((nrows + T - 1) / T);
  return launch_pass<LOGL, T, MODE_ROW, FWD>(ctx, io, grid, 0);
}

// ---- tensor maps for the TMA-fed passes --------------------------------------------------------
typedef CUresult (*encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static encode_tiled_fn get_encode_tiled() {
  // resolved once; function-local static initialisation is thread-safe (contexts may be driven from several threads)
  static const encode_tiled_fn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      return reinterpret_cast<encode_tiled_fn>(p);
    return static_cast<encode_tiled_fn>(nullptr);
  }();
  return fn;
}

// complex64 elements are described to TMA as 8-byte integers; dims/box are innermost first
static bool make_tensor_map(tensor_map_blob* out, const void* base, int rank, const cuuint64_t* dims,
                            const cuuint64_t* strides_bytes /* rank-1 */, const cuuint32_t* box,
                            CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_INT64,
                            CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_NONE) {
  encode_tiled_fn enc = get_encode_tiled();
  if (!enc) return false;
  static_assert(sizeof(CUtensorMap) <= sizeof(tensor_map_blob), "tensor map size");
  cuuint32_t estr[3] = {1, 1, 1};
  CUtensorMap m;
  const CUresult r = enc(&m, dtype, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes,
                         box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return false;
  std::memcpy(out->bytes, &m, sizeof(m));
  return true;
}

// three-sweep factorisation of 2^q: the first sweep takes ceil(q/3); of the rest the longer half goes to the
// LAST sweep (2^23 = 2^8 * 2^7 * 2^8) so that the transposing pass runs as 16 x 16
static void plan3(int q, int* l1, int* l2, int* l3) {
  *l1 = (q + 2) / 3;
  const int big = (q - *l1 + 1) / 2, small = q - *l1 - big;
  // the fused R2C last sweep exists up to L = 256: keep the last factor <= 8 when one of the two is
  const bool last_big = big <= 8;
  *l2 = last_big ? small : big;
  *l3 = last_big ? big : small;
}

// 2^27 points and above: four sweeps of L <= 256 (all on the sixteen-point kernels, each near the HBM roofline)
// beat three sweeps with 512/1024-point columns; the last factor is 7 or 8 so the fused R2C last sweep applies.
// 27 = 7+7+6+7, 28 = 7+7+7+7, 29 = 7+7+7+8, 30 = 8+7+7+8. Unaligned data or no TMA keeps three sweeps.
static void plan4(int q, int* l) {
  l[3] = (q >= 29) ? 8 : 7;
  int r = q - l[3];
  l[0] = (r + 2) / 3;
  l[1] = (r - l[0] + 1) / 2;
  l[2] = r - l[0] - l[1];
}
static bool four_sweeps(int q, const void* ptr) {
  return q >= 27 && q <= 30 && get_encode_tiled() != nullptr && (reinterpret_cast<uintptr_t>(ptr) & 15u) == 0;
}

// wide tiles (32 neighbouring columns = 256-byte segments) for the 128-point column sweep of very long transforms,
// whose row stride is megabytes: fewer DRAM page openings / TLB entries per byte
static bool wide_col(size_t A, size_t L, size_t B) {
  return B >= ((size_t)1 << 14) && A * L * B >= ((size_t)1 << 26);
}

template <int LOGL, bool FWD, int TT = col_t<LOGL>::value>
static int launch_col_tma(srtb_b200_ctx* ctx, const float2* in, float2* out, size_t A, size_t B, bool* done,
                          const row_chirp_params* chirp = nullptr) {
  constexpr int T = TT, L = 1 << LOGL;
  if constexpr (LOGL == 7 && TT == col_t<LOGL>::value) {
    if (wide_col(A, L, B) && !chirp) return launch_col_tma<LOGL, FWD, 32>(ctx, in, out, A, B, done);
  }
  *done = false;
  if ((reinterpret_cast<uintptr_t>(in) & 15u) || A * L >= ((size_t)1 << 31) || B >= ((size_t)1 << 31)) return 0;
  tensor_map_blob tm;
  const cuuint64_t dims[2] = {(cuuint64_t)B, (cuuint64_t)(A * L)};
  const cuuint64_t strides[1] = {(cuuint64_t)B * sizeof(float2)};
  const cuuint32_t box[2] = {(cuuint32_t)T, (cuuint32_t)std::min(L, 256)};
  if (!make_tensor_map(&tm, in, 2, dims, strides, box)) return 0;  // fall back to the LDG kernel
  big_twiddle btw;
  if (int rc = get_big_twiddles(ctx, LOGL + ilog2(B), &btw)) return rc;
  const float2* tw = nullptr;
  if (int rc = get_stage_twiddles(ctx, LOGL, &tw)) return rc;
  const size_t smem = tile_tma_smem<LOGL, T>::bytes(btw.q);
  const size_t ntiles = A * (B / T);
  unsigned grid = 1;
  if constexpr (LOGL >= 7 && LOGL <= 9) {
    auto kern16 = fft_col16_tma_kernel<LOGL, T, FWD>;
    constexpr int threads = col16_threads<LOGL, T>::value;
    const size_t smem16 = col16_smem<LOGL, T, false>::bytes(btw.q);
    if (int rc = persistent_grid(ctx, kern16, threads, smem16, col16_smem<LOGL, T, false>::bytes(10), ntiles, &grid)) return rc;
    if constexpr (!FWD && LOGL >= 8) {
      if (chirp) {  // s1 + chirp applied as the tile is read (long waterfall rows: a 2^8 or 2^9 first sweep)
        auto kernc = fft_col16_tma_kernel<LOGL, T, FWD, 0, true>;
        if (int rc = persistent_grid(ctx, kernc, threads, smem, tile_tma_smem<LOGL, T>::bytes(10), ntiles, &grid)) return rc;
        CK(launch(ctx, true, kernc, grid, threads, smem, tm, out, B, (uint32_t)(B / T), (uint32_t)ntiles, btw, tw,
                  raw_params{}, *chirp));
        *done = true;
        return 0;
      }
    } else {
      if (chirp) return 0;  // no chirp-on-load kernel for a 2^7 column sweep (nor for a forward one)
    }
    CK(launch(ctx, true, kern16, grid, threads, smem16, tm, out, B, (uint32_t)(B / T), (uint32_t)ntiles, btw, tw,
              raw_params{}, row_chirp_params{}));
  } else {
    if (chirp) return 0;  // the chirp-on-load sweep exists for the sixteen-point kernel only
    auto kern = fft_col_tma_kernel<LOGL, T, FWD>;
    if (int rc = persistent_grid(ctx, kern, pass_threads<LOGL, T>::value, smem, tile_tma_smem<LOGL, T>::bytes(10), ntiles, &grid)) return rc;
    CK(launch(ctx, false, kern, grid, pass_threads<LOGL, T>::value, smem, tm, out, B, (uint32_t)(B / T), (uint32_t)ntiles,
              btw, tw));
  }
  *done = true;
  return 0;
}

// first pass of the packed real transform straight from the 8-bit baseband (unpack fused in)
struct raw_source {
  const void* base = nullptr;  // device pointer to the block's bytes
  int G = 0, o0 = 0, o1 = 0;   // bytes per complex point, byte offsets of its two samples
  int delta = 0;               // subtracted from the offsets of odd points (gznupsr_a1 word layout)
  int bits = 0;                // 2 or 4: packed unsigned samples (G, o0, o1 unused)
  bool is_signed = true;
};

// the first sweep of the packed R2C plans that take the raw route is 2^7 .. 2^9 points long (plan3 / plan4 on a
// 16-byte aligned buffer; the two-sweep plans with a first sweep of 2^10 end on a 2^9 or 2^10 last sweep, which has no
// fused R2C split), or 2^11 on the sweep-order route of 2^25-point blocks (r2c_sweep_order)
template <int LOGL, int RAW, int TT = col_t<LOGL>::value>
static int launch_col_tma_raw(srtb_b200_ctx* ctx, const raw_source& src, float2* out, size_t B, bool* done) {
  static_assert((LOGL >= 7 && LOGL <= 9) || LOGL == 11, "raw first sweep: sixteen-point column kernel only");
  constexpr int T = TT, L = 1 << LOGL;
  if constexpr (LOGL == 7 && TT == col_t<LOGL>::value) {
    if (wide_col(1, L, B)) return launch_col_tma_raw<LOGL, RAW, 32>(ctx, src, out, B, done);
  }
  *done = false;
  if ((reinterpret_cast<uintptr_t>(src.base) & 15u) || B >= ((size_t)1 << 29)) return 0;
  // one tile row = T complex points: T * G bytes, or T * bits / 4 bytes of packed samples; TMA wants >= 16 bytes
  const size_t row_bytes = (RAW == 3) ? (size_t)T * src.bits / 4 : (size_t)T * src.G;
  const size_t line_bytes = (RAW == 3) ? B * src.bits / 4 : B * src.G;
  if (row_bytes < 16 || (row_bytes & 15) || (line_bytes & 15) || row_bytes > (size_t)T * 4) return 0;
  tensor_map_blob tm;
  const cuuint64_t dims[2] = {(cuuint64_t)line_bytes, (cuuint64_t)L};
  const cuuint64_t strides[1] = {(cuuint64_t)line_bytes};
  const cuuint32_t box[2] = {(cuuint32_t)row_bytes, (cuuint32_t)std::min(L, 256)};
  if (!make_tensor_map(&tm, src.base, 2, dims, strides, box, CU_TENSOR_MAP_DATA_TYPE_UINT8)) return 0;
  big_twiddle btw;
  if (int rc = get_big_twiddles(ctx, LOGL + ilog2(B), &btw)) return rc;
  const float2* tw = nullptr;
  if (int rc = get_stage_twiddles(ctx, LOGL, &tw)) return rc;
  const size_t smem = tile_tma_smem<LOGL, T>::bytes(btw.q);
  const size_t ntiles = B / T;
  unsigned grid = 1;
  const raw_params rp{src.G, src.o0, src.o1, src.delta, (int)row_bytes, src.bits};
  constexpr int threads = col16_threads<LOGL, T>::value;
  constexpr size_t smem16 = raw16_smem<LOGL, T>::bytes;  // inter-sweep tables stay in global memory here
  if constexpr (LOGL == 11) {
    static_assert(T == 8, "the 2^11-point raw sweep has 32-byte raw rows and 64-byte stores");
    auto kern = r2c_raw_col2048_kernel<RAW>;
    if (int rc = persistent_grid(ctx, kern, threads, smem16, smem16, ntiles, &grid)) return rc;
    CK(launch(ctx, true, kern, grid, threads, smem16, tm, out, B, (uint32_t)(B / T), (uint32_t)ntiles, btw, tw, rp));
  } else {
    auto kern16 = fft_col16_tma_kernel<LOGL, T, true, RAW>;
    if (int rc = persistent_grid(ctx, kern16, threads, smem16, smem16, ntiles, &grid)) return rc;
    CK(launch(ctx, true, kern16, grid, threads, smem16, tm, out, B, (uint32_t)(B / T), (uint32_t)ntiles, btw, tw, rp,
              row_chirp_params{}));
  }
  *done = true;
  return 0;
}

static int dispatch_col_raw(srtb_b200_ctx* ctx, int logl, const raw_source& src, float2* out, size_t B, bool* done) {
  *done = false;
  if (src.bits) {  // packed 2- / 4-bit samples
    switch (logl) {
      case 7: return launch_col_tma_raw<7, 3>(ctx, src, out, B, done);
      case 8: return launch_col_tma_raw<8, 3>(ctx, src, out, B, done);
      default: return 0;
    }
  }
  switch (logl) {
    case 7: return src.is_signed ? launch_col_tma_raw<7, 1>(ctx, src, out, B, done) : launch_col_tma_raw<7, 2>(ctx, src, out, B, done);
    case 8: return src.is_signed ? launch_col_tma_raw<8, 1>(ctx, src, out, B, done) : launch_col_tma_raw<8, 2>(ctx, src, out, B, done);
    case 9: return src.is_signed ? launch_col_tma_raw<9, 1>(ctx, src, out, B, done) : launch_col_tma_raw<9, 2>(ctx, src, out, B, done);
    case 11: return src.is_signed ? launch_col_tma_raw<11, 1>(ctx, src, out, B, done) : launch_col_tma_raw<11, 2>(ctx, src, out, B, done);
    default: return 0;
  }
}

template <int LOGL, bool FWD>
static int launch_trans_tma(srtb_b200_ctx* ctx, const float2* in, float2* out, size_t batch, size_t A, size_t L1,
                            bool* done, size_t rest_inner = 0, float2* tile_stats = nullptr) {
  constexpr int T = col_t<LOGL>::value, L = 1 << LOGL;
  *done = false;
  const size_t S = A / L1;
  if ((reinterpret_cast<uintptr_t>(in) & 15u) || batch * L1 >= ((size_t)1 << 31)) return 0;
  tensor_map_blob tm;
  // rows [beta*L1 + k1][rest][L]  ->  dims (L, S, batch*L1)
  const cuuint64_t dims[3] = {(cuuint64_t)L, (cuuint64_t)S, (cuuint64_t)(batch * L1)};
  const cuuint64_t strides[2] = {(cuuint64_t)L * sizeof(float2), (cuuint64_t)S * L * sizeof(float2)};
  const cuuint32_t box[3] = {(cuuint32_t)std::min(L, 256), 1u, (cuuint32_t)((L <= 256) ? T : 1)};
  if (!make_tensor_map(&tm, in, 3, dims, strides, box)) return 0;
  const float2* tw = nullptr;
  if (int rc = get_stage_twiddles(ctx, LOGL, &tw)) return rc;
  const size_t smem = tile_tma_smem<LOGL, T>::bytes(0);
  const size_t k1tiles = L1 / T, ntiles = batch * S * k1tiles;
  unsigned grid = 1;
  if constexpr (LOGL == 7 || LOGL == 8) {
    auto kern16 = fft_trans16_tma_kernel<LOGL, T, FWD>;
    constexpr int threads = T * (L / 16);
    if (int rc = persistent_grid(ctx, kern16, threads, smem, smem, ntiles, &grid)) return rc;
    CK(launch(ctx, false, kern16, grid, threads, smem, tm, out, (uint32_t)A, (uint32_t)S, (uint32_t)L1, (uint32_t)k1tiles,
              (uint32_t)ntiles, tw, (uint32_t)rest_inner, tile_stats));
  } else {
    if (rest_inner > 1) return 0;  // only the sixteen-point kernel knows the four-sweep row order
    auto kern = fft_trans_tma_kernel<LOGL, T, FWD>;
    if (int rc = persistent_grid(ctx, kern, pass_threads<LOGL, T>::value, smem, smem, ntiles, &grid)) return rc;
    CK(launch(ctx, false, kern, grid, pass_threads<LOGL, T>::value, smem, tm, out, (uint32_t)A, (uint32_t)S, (uint32_t)L1,
              (uint32_t)k1tiles, (uint32_t)ntiles, tw, tile_stats));
  }
  *done = true;
  return 0;
}

template <int LOGL, bool FWD>
static int launch_col(srtb_b200_ctx* ctx, const float2* in, float2* out, size_t A, size_t B) {
  constexpr int T = col_t<LOGL>::value;
  {
    bool done = false;
    if (int rc = launch_col_tma<LOGL, FWD>(ctx, in, out, A, B, &done)) return rc;
    if (done) return 0;
  }
  col_io<LOGL, T, FWD> io;
  io.in = in;
  io.out = out;
  io.B = B;
  io.btiles = (uint32_t)(B / T);
  if (int rc = get_big_twiddles(ctx, LOGL + ilog2(B), &io.btw)) return rc;
  io.base = 0;
  io.b0 = 0;
  io.stw = nullptr;
  const unsigned grid = (unsigned)(A * (B / T));
  return launch_pass<LOGL, T, MODE_COL, FWD>(ctx, io, grid, (size_t)(3u << io.btw.q) * sizeof(float2));
}

template <int LOGL, bool FWD>
static int launch_trans(srtb_b200_ctx* ctx, const float2* in, float2* out, size_t batch, size_t A,
                        size_t L1) {
  constexpr int T = col_t<LOGL>::value;
  {
    bool done = false;
    if (int rc = launch_trans_tma<LOGL, FWD>(ctx, in, out, batch, A, L1, &done)) return rc;
    if (done) return 0;
  }
  trans_io<LOGL, T> io;
  io.in = in;
  io.out = out;
  io.A = (uint32_t)A;
  io.S = (uint32_t)(A / L1);
  io.L1 = (uint32_t)L1;
  io.k1tiles = (uint32_t)(L1 / T);
  io.in_row0 = 0;
  io.out0 = 0;
  const unsigned grid = (unsigned)(batch * io.S * io.k1tiles);
  return launch_pass<LOGL, T, MODE_TRANS, FWD>(ctx, io, grid, 0);
}

#define SRTB_DISPATCH_LOGL(fn, logl, lo, hi, ...)                       \
  switch (logl) {                                                       \
    case 3: if (lo <= 3 && 3 <= hi) return fn<(lo <= 3 && 3 <= hi) ? 3 : lo, FWD>(__VA_ARGS__); break;   \
    case 4: if (lo <= 4 && 4 <= hi) return fn<(lo <= 4 && 4 <= hi) ? 4 : lo, FWD>(__VA_ARGS__); break;   \
    case 5: if (lo <= 5 && 5 <= hi) return fn<(lo <= 5 && 5 <= hi) ? 5 : lo, FWD>(__VA_ARGS__); break;   \
    case 6: if (lo <= 6 && 6 <= hi) return fn<(lo <= 6 && 6 <= hi) ? 6 : lo, FWD>(__VA_ARGS__); break;   \
    case 7: if (lo <= 7 && 7 <= hi) return fn<(lo <= 7 && 7 <= hi) ? 7 : lo, FWD>(__VA_ARGS__); break;   \
    case 8: if (lo <= 8 && 8 <= hi) return fn<(lo <= 8 && 8 <= hi) ? 8 : lo, FWD>(__VA_ARGS__); break;   \
    case 9: if (lo <= 9 && 9 <= hi) return fn<(lo <= 9 && 9 <= hi) ? 9 : lo, FWD>(__VA_ARGS__); break;   \
    case 10: if (lo <= 10 && 10 <= hi) return fn<(lo <= 10 && 10 <= hi) ? 10 : lo, FWD>(__VA_ARGS__); break; \
    case 11: if (lo <= 11 && 11 <= hi) return fn<(lo <= 11 && 11 <= hi) ? 11 : lo, FWD>(__VA_ARGS__); break; \
    case 12: if (lo <= 12 && 12 <= hi) return fn<(lo <= 12 && 12 <= hi) ? 12 : lo, FWD>(__VA_ARGS__); break; \
    default: break;                                                     \
  }

template <bool FWD>
static int dispatch_row(srtb_b200_ctx* ctx, int logl, const float2* in, float2* out, size_t nrows) {
  SRTB_DISPATCH_LOGL(launch_row, logl, 3, 12, ctx, in, out, nrows)
  return fail(ctx, SRTB_B200_E_SIZE, "fft: unsupported row length 2^" + std::to_string(logl));
}
template <bool FWD>
static int dispatch_col(srtb_b200_ctx* ctx, int logl, const float2* in, float2* out, size_t A, size_t B) {
  SRTB_DISPATCH_LOGL(launch_col, logl, 6, 10, ctx, in, out, A, B)
  return fail(ctx, SRTB_B200_E_SIZE, "fft: unsupported column length 2^" + std::to_string(logl));
}
template <bool FWD>
static int dispatch_trans(srtb_b200_ctx* ctx, int logl, const float2* in, float2* out, size_t batch,
                          size_t A, size_t L1) {
  SRTB_DISPATCH_LOGL(launch_trans, logl, 6, 10, ctx, in, out, batch, A, L1)
  return fail(ctx, SRTB_B200_E_SIZE, "fft: unsupported last-pass length 2^" + std::to_string(logl));
}

// ---- whole-row waterfall kernel (fft_bigrow.cuh): rows of 2^13 / 2^14 points held in one CTA's shared memory.
// Unaligned rows of these lengths take the two-sweep column + transposing plan.

template <int LOGL>
static int get_bigrow_tables(srtb_b200_ctx* ctx, bool fwd, const float2** out) {
  using C = bigrow<LOGL>;
  buffer<float2>& d = ctx->bigrow_tab[LOGL - 13][fwd ? 1 : 0];
  if (!d.p) {
    std::vector<float2> h(C::TABN);
    const double sgn = fwd ? -1.0 : 1.0;
    auto w = [&](size_t n, size_t e) {
      const double a = sgn * 2.0 * M_PI * (double)(e % n) / (double)n;
      return make_float2((float)std::cos(a), (float)std::sin(a));
    };
    for (int j = 0; j < C::B1; j++) h[j] = w(C::L, j);
    for (int i = 1; i < 16; i++)
      for (int j = 0; j < C::B2; j++) h[C::B1 + (i - 1) * C::B2 + j] = w(C::B1, (size_t)i * j);
    for (int i = 1; i < 16; i++)
      for (int j = 0; j < C::R3; j++) h[C::B1 + 15 * C::B2 + (i - 1) * C::R3 + j] = w(C::B2, (size_t)i * j);
    if (int rc = upload_table(ctx, h, &d)) return rc;
  }
  *out = d.p;
  return 0;
}

// sk != nullptr: SK + column sums in the epilogue (sk->partial is filled in here); chirp != nullptr: s1 + chirp on load.
// sweep_order: `in` is the channel-blocked spectrum r2c_sweep_order leaves (P = nrows = L / 8), read channel by channel
template <int LOGL, bool FWD>
static int launch_bigrow(srtb_b200_ctx* ctx, const float2* in, float2* out, size_t nrows, row_sk_params* sk,
                         const row_chirp_params* chirp, size_t* chunks_out, bool sweep_order = false) {
  using C = bigrow<LOGL>;
  if (nrows >= ((size_t)1 << 31)) return fail(ctx, SRTB_B200_E_SIZE, "fft: too many rows");
  const float2* tabs = nullptr;
  if (int rc = get_bigrow_tables<LOGL>(ctx, FWD, &tabs)) return rc;
  unsigned grid = 1;
  auto go = [&](auto kern, bool with_sk, auto... extra) -> int {
    const size_t smem = sweep_order ? C::bytes_sw : C::bytes;
    if (int rc = persistent_grid(ctx, kern, C::NT, smem, smem, nrows, &grid)) return rc;
    row_sk_params p{};
    if (with_sk) {
      if (int rc = grow(ctx, ctx->lane.colsum_partial, (size_t)grid * sk->ts_count * sizeof(float))) return rc;
      sk->partial = ctx->lane.colsum_partial.p;
      p = *sk;
    }
    CK(launch(ctx, true, kern, grid, C::NT, smem, in, out, (unsigned)nrows, tabs, p, chirp ? *chirp : row_chirp_params{},
              extra...));
    if (chunks_out) *chunks_out = grid;
    return 0;
  };
  if constexpr (!FWD && LOGL == 14) {
    if (sweep_order) {
      if (!(sk && chirp && chirp->newton == 2) || nrows * 8 != (size_t)C::L)
        return fail(ctx, SRTB_B200_E_UNSUPPORTED, "watfft: the sweep-order load needs the exact chirp and P = L / 8");
      // the spectrum as lines of 16 elements (128 bytes); a box is a quarter of a half channel, 128 lines, swizzled so
      // that stage 0's gather is conflict free without moving registers around
      const cuuint64_t dims[2] = {16u, (cuuint64_t)nrows * C::L / 16};
      const cuuint64_t strides[1] = {16 * sizeof(float2)};
      const cuuint32_t box[2] = {16u, 128u};
      tensor_map_blob tm;
      if (!make_tensor_map(&tm, in, 2, dims, strides, box, CU_TENSOR_MAP_DATA_TYPE_INT64, CU_TENSOR_MAP_SWIZZLE_128B))
        return fail(ctx, SRTB_B200_E_UNSUPPORTED, "watfft: tensor map of the sweep-order spectrum refused");
      return go(waterfall_sweep_order_kernel, true, tm);
    }
  }
  if (sweep_order) return fail(ctx, SRTB_B200_E_UNSUPPORTED, "watfft: sweep-order load exists for rows of 2^14");
  if constexpr (!FWD) {
    if (sk && chirp && chirp->newton == 5) return go(fft_bigrow_kernel<LOGL, false, true, 5>, true);
    if (sk && chirp && chirp->newton == 1) return go(fft_bigrow_kernel<LOGL, false, true, 1>, true);
    if (sk && chirp && chirp->newton == 3) return go(fft_bigrow_kernel<LOGL, false, true, 3>, true);
    if (sk && chirp && chirp->newton == 4) return go(fft_bigrow_kernel<LOGL, false, true, 4>, true);
    if (sk && chirp) return go(fft_bigrow_kernel<LOGL, false, true, 2>, true);
  }
  if (sk || chirp) return fail(ctx, SRTB_B200_E_UNSUPPORTED, "fft: fused epilogue exists for the backward transform with the chirp only");
  return go(fft_bigrow_kernel<LOGL, FWD, false, 0>, false);
}

// the R2C row sweep of the sweep-order route: P rows of 2^14 points of the scratch s (clusters of two CTAs), the
// spectrum channel-blocked to out, leaving mean(|X_k|^2, k < M) in the lane's `mean`
static int launch_r2c_rows(srtb_b200_ctx* ctx, const float2* s, float2* out, size_t P) {
  using C = bigrow<14>;
  auto kern = r2c_rows_split_kernel;
  const float2* tabs = nullptr;
  if (int rc = get_bigrow_tables<14>(ctx, true, &tabs)) return rc;
  cudaLaunchConfig_t cfg{};
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.blockDim = dim3(C::NT);
  cfg.dynamicSmemBytes = C::bytes_r2c;
  cfg.stream = ctx->lane.stream;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (int rc = set_smem_max(ctx, kern, C::bytes_r2c)) return rc;
  const void* key = reinterpret_cast<const void*>(kern);
  if (!ctx->occupancy.count(key)) {
    int clusters = 0;
    cfg.gridDim = dim3(2 * (unsigned)ctx->sm_count);
    CK(cudaOccupancyMaxActiveClusters(&clusters, kern, &cfg));
    if (clusters < 1) return fail(ctx, SRTB_B200_E_UNSUPPORTED, "r2c: no two-CTA cluster of the row sweep fits an SM pair");
    ctx->occupancy[key] = clusters;
  }
  const unsigned clusters = (unsigned)std::min<size_t>(P / 2, (size_t)ctx->occupancy[key]);
  if (2 * clusters > 4096) return fail(ctx, SRTB_B200_E_SIZE, "r2c: partial buffer too small");
  cfg.gridDim = dim3(2 * clusters);
  cfg.numAttrs = ctx->pdl_auto ? 2 : 1;
  CK(launch(ctx, cfg, kern, s, out, (unsigned)P, tabs, r2c_rows_params{ctx->lane.partial, ctx->lane.ticket, ctx->lane.mean}));
  return 0;
}

// L = 2 or 4: one thread per row
template <bool FWD>
__global__ void tiny_fft_kernel(float2* x, int logl, size_t nrows) {
  const size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nrows) return;
  if (logl == 1) {
    float2 a = x[2 * r], b = x[2 * r + 1];
    dft2<FWD>(a, b);
    x[2 * r] = a;
    x[2 * r + 1] = b;
  } else {
    float2 a = x[4 * r], b = x[4 * r + 1], c = x[4 * r + 2], d = x[4 * r + 3];
    dft4<FWD>(a, b, c, d);
    x[4 * r] = a;
    x[4 * r + 1] = b;
    x[4 * r + 2] = c;
    x[4 * r + 3] = d;
  }
}

template <bool FWD>
static int fft_c2c_impl(srtb_b200_ctx* ctx, float2* x, size_t n, size_t batch) {
  const int q = ilog2(n);
  if (q == 0) return 0;
  if (q <= 2) {
    CK(launch(ctx, false, tiny_fft_kernel<FWD>, (unsigned)((batch + 255) / 256), 256, 0, x, q, batch));
    return 0;
  }
  if (q <= 12) return dispatch_row<FWD>(ctx, q, x, x, batch);
  if ((q == 13 || q == 14) && (reinterpret_cast<uintptr_t>(x) & 15u) == 0) {
    // one sweep: the whole row in shared memory (in place: a CTA reads its row completely before it stores it)
    return q == 13 ? launch_bigrow<13, FWD>(ctx, x, x, batch, nullptr, nullptr, nullptr)
                   : launch_bigrow<14, FWD>(ctx, x, x, batch, nullptr, nullptr, nullptr);
  }
  if (q > 30) return fail(ctx, SRTB_B200_E_SIZE, "fft: length above 2^30 not supported");
  if (int rc = grow(ctx, ctx->lane.fft_scratch, batch * n * sizeof(float2))) return rc;
  float2* s = ctx->lane.fft_scratch.p;
  if (q <= 20) {
    const int l1 = (q + 1) / 2, l2 = q - l1;
    const size_t L1 = (size_t)1 << l1, L2 = (size_t)1 << l2;
    if (int rc = dispatch_col<FWD>(ctx, l1, x, s, batch, L2)) return rc;
    return dispatch_trans<FWD>(ctx, l2, s, x, batch, L1, L1);
  }
  if (four_sweeps(q, x)) {
    int l[4];
    plan4(q, l);
    const size_t L1 = (size_t)1 << l[0], L2 = (size_t)1 << l[1], L3 = (size_t)1 << l[2];
    const size_t L4 = (size_t)1 << l[3];
    if (int rc = dispatch_col<FWD>(ctx, l[0], x, s, batch, L2 * L3 * L4)) return rc;
    if (int rc = dispatch_col<FWD>(ctx, l[1], s, s, batch * L1, L3 * L4)) return rc;
    if (int rc = dispatch_col<FWD>(ctx, l[2], s, s, batch * L1 * L2, L4)) return rc;
    bool done = false;
    int rc = (l[3] == 7) ? launch_trans_tma<7, FWD>(ctx, s, x, batch, L1 * L2 * L3, L1, &done, L3)
                         : launch_trans_tma<8, FWD>(ctx, s, x, batch, L1 * L2 * L3, L1, &done, L3);
    if (rc) return rc;
    if (!done) return fail(ctx, SRTB_B200_E_UNSUPPORTED, "fft: four-sweep plan needs the TMA last sweep");
    return 0;
  }
  int l1, l2, l3;
  plan3(q, &l1, &l2, &l3);
  const size_t L1 = (size_t)1 << l1, L2 = (size_t)1 << l2, L3 = (size_t)1 << l3;
  if (int rc = dispatch_col<FWD>(ctx, l1, x, s, batch, L2 * L3)) return rc;
  if (int rc = dispatch_col<FWD>(ctx, l2, s, s, batch * L1, L3)) return rc;
  return dispatch_trans<FWD>(ctx, l3, s, x, batch, L1 * L2, L1);
}

extern "C" int srtb_b200_fft_c2c(srtb_b200_ctx* ctx, void* d_x, size_t length, size_t batch, int direction) {
  API_LOCK(ctx);
  if (!ctx || !d_x) return fail(ctx, SRTB_B200_E_INVALID, "fft_c2c: null argument");
  if (!aligned8(d_x)) return fail(ctx, SRTB_B200_E_INVALID, "fft_c2c: d_x is not 8-byte aligned");
  if (length == 0 || batch == 0) return fail(ctx, SRTB_B200_E_INVALID, "fft_c2c: zero size");
  if (!is_pow2(length))
    return fail(ctx, SRTB_B200_E_SIZE, "[fft] n must be a power of 2, got " + std::to_string(length));
  if (length > ((size_t)1 << 30)) return fail(ctx, SRTB_B200_E_SIZE, "fft: length above 2^30 not supported");
  if (batch > ((size_t)1 << 34) / length) return fail(ctx, SRTB_B200_E_SIZE, "fft: batch * length above 2^34");
  if (direction != 1 && direction != -1) return fail(ctx, SRTB_B200_E_INVALID, "fft_c2c: direction must be +1 / -1");
  CK(cudaSetDevice(ctx->device));
  if (direction == 1) return fft_c2c_impl<true>(ctx, static_cast<float2*>(d_x), length, batch);
  return fft_c2c_impl<false>(ctx, static_cast<float2*>(d_x), length, batch);
}

extern "C" int srtb_b200_watfft_c2c_backward(srtb_b200_ctx* ctx, void* d_x, size_t length, size_t batch) {
  API_LOCK(ctx);
  if (!ctx) return fail(nullptr, SRTB_B200_E_INVALID, "watfft: ctx is null");
  if (!aligned8(d_x)) return fail(ctx, SRTB_B200_E_INVALID, "watfft: d_x is not 8-byte aligned");
  stage_scope stats_(ctx, SRTB_B200_STAGE_WATFFT, 16.0 * (double)length * (double)batch);
  return srtb_b200_fft_c2c(ctx, d_x, length, batch, -1);
}

static int fft_r2c_with_power_mean(srtb_b200_ctx* ctx, float* d_inout, size_t n_real, const raw_source* raw = nullptr,
                                   bool* raw_used = nullptr);

extern "C" int srtb_b200_fft_r2c_inplace(srtb_b200_ctx* ctx, float* d_inout, size_t n_real) {
  API_LOCK(ctx);
  if (!ctx || !d_inout) return fail(ctx, SRTB_B200_E_INVALID, "fft_r2c: null argument");
  if (!aligned8(d_inout)) return fail(ctx, SRTB_B200_E_INVALID, "fft_r2c: d_inout is not 8-byte aligned");
  if (n_real < 2 || !is_pow2(n_real))
    return fail(ctx, SRTB_B200_E_SIZE, "[fft] n must be a power of 2, got " + std::to_string(n_real));
  CK(cudaSetDevice(ctx->device));
  const size_t M = n_real / 2;
  stage_scope stats_(ctx, SRTB_B200_STAGE_FFT_R2C, 8.0 * (double)n_real);
  if (M >= ((size_t)1 << 13) && (reinterpret_cast<uintptr_t>(d_inout) & 15u) == 0)
    return fft_r2c_with_power_mean(ctx, d_inout, n_real);  // multi-sweep sizes: split fused into the last sweep
  float2* H = reinterpret_cast<float2*>(d_inout);
  if (int rc = fft_c2c_impl<true>(ctx, H, M, 1)) return rc;
  CK(launch(ctx, false, r2c_post_kernel<false>, grid_for(ctx, M / 2 + 1, 256), 256, 0, H, M, nullptr, nullptr, nullptr));
  return 0;
}

// launch of the fused last pass + split (LOGL <= 8 keeps two [2T][L] tiles double-buffered in smem)
template <int LOGL>
static int launch_trans_r2c(srtb_b200_ctx* ctx, const float2* in, float2* out, size_t A, size_t L1, bool* done,
                            size_t rest_inner = 0) {
  constexpr int T = 8, L = 1 << LOGL;
  *done = false;
  const size_t S = A / L1;
  if ((reinterpret_cast<uintptr_t>(in) & 15u) || L1 < 4 * T || L1 >= ((size_t)1 << 31)) return 0;
  tensor_map_blob tm;
  const cuuint64_t dims[3] = {(cuuint64_t)L, (cuuint64_t)S, (cuuint64_t)L1};
  const cuuint64_t strides[2] = {(cuuint64_t)L * sizeof(float2), (cuuint64_t)S * L * sizeof(float2)};
  const cuuint32_t box[3] = {(cuuint32_t)L, 1u, (cuuint32_t)T};
  if (!make_tensor_map(&tm, in, 3, dims, strides, box)) return 0;
  const float2* tw = nullptr;
  if (int rc = get_stage_twiddles(ctx, LOGL, &tw)) return rc;
  constexpr size_t smem = trans_r2c_smem<LOGL, T>::bytes;
  const size_t tiles_per_rest = L1 / (2 * T) + 1, ntiles = S * tiles_per_rest;
  unsigned grid = 1;
  if constexpr (LOGL == 7 || LOGL == 8) {
    auto kern16 = fft_trans_r2c16_tma_kernel<LOGL, T>;
    constexpr int threads = 2 * T * (L / 16);
    if (int rc = persistent_grid(ctx, kern16, threads, smem, smem, ntiles, &grid)) return rc;
    grid = std::min<unsigned>(grid, 2048);
    CK(launch(ctx, true, kern16, grid, threads, smem, tm, out, (uint32_t)A, (uint32_t)S, (uint32_t)L1,
              (uint32_t)tiles_per_rest, (uint32_t)ntiles, tw, ctx->lane.partial, (uint32_t)rest_inner));
  } else {
    if (rest_inner > 1) return 0;  // four-sweep row order: sixteen-point kernel only
    auto kern = fft_trans_r2c_tma_kernel<LOGL, T>;
    if (int rc = persistent_grid(ctx, kern, 2 * pass_threads<LOGL, T>::value, smem, smem, ntiles, &grid)) return rc;
    grid = std::min<unsigned>(grid, 2048);
    CK(launch(ctx, false, kern, grid, 2 * pass_threads<LOGL, T>::value, smem, tm, out, (uint32_t)A, (uint32_t)S,
              (uint32_t)L1, (uint32_t)tiles_per_rest, (uint32_t)ntiles, tw, ctx->lane.partial));
  }
  {
    const size_t pairs = ((A << LOGL) / L1) / 2 + 1;
    const unsigned fgrid = (unsigned)std::min<size_t>((pairs + 255) / 256, 2048);
    if (grid + fgrid > 4096) return fail(ctx, SRTB_B200_E_SIZE, "r2c: partial buffer too small");
    CK(launch(ctx, true, r2c_col0_fixup_kernel, fgrid, 256, 0, out, (size_t)(A << LOGL), (size_t)L1, ctx->lane.partial,
              (unsigned)grid, ctx->lane.ticket, ctx->lane.mean));
  }
  *done = true;
  return 0;
}

// R2C whose split pass also leaves mean(|X_k|^2, k < N/2) in ctx->lane.mean (used by process_block:
// the s1 statistic costs no extra sweep). For multi-pass sizes the split is fused into the last FFT
// pass (fft_trans_r2c_tma_kernel), so the packed transform costs P sweeps instead of P + 1.
static int fft_r2c_with_power_mean(srtb_b200_ctx* ctx, float* d_inout, size_t n_real, const raw_source* raw,
                                   bool* raw_used) {
  if (raw_used) *raw_used = false;
  const size_t M = n_real / 2;
  float2* H = reinterpret_cast<float2*>(d_inout);
  const int q = ilog2(M);
  if (q >= 13 && q <= 30 && M >= 2) {
    // same factorisation as fft_c2c_impl
    if (four_sweeps(q, d_inout)) {
      int l[4];
      plan4(q, l);
      if (int rc = grow(ctx, ctx->lane.fft_scratch, M * sizeof(float2))) return rc;
      float2* s = ctx->lane.fft_scratch.p;
      const size_t L1 = (size_t)1 << l[0], L2 = (size_t)1 << l[1], L3 = (size_t)1 << l[2], L4 = (size_t)1 << l[3];
      bool first_done = false;
      if (raw && raw->base) {
        if (int rc = dispatch_col_raw(ctx, l[0], *raw, s, L2 * L3 * L4, &first_done)) return rc;
        if (raw_used) *raw_used = first_done;
        if (!first_done) return SRTB_B200_E_UNSUPPORTED;
      }
      if (!first_done)
        if (int rc = dispatch_col<true>(ctx, l[0], H, s, 1, L2 * L3 * L4)) return rc;
      if (int rc = dispatch_col<true>(ctx, l[1], s, s, L1, L3 * L4)) return rc;
      if (int rc = dispatch_col<true>(ctx, l[2], s, s, L1 * L2, L4)) return rc;
      bool done = false;
      int rc = (l[3] == 7) ? launch_trans_r2c<7>(ctx, s, H, L1 * L2 * L3, L1, &done, L3)
                           : launch_trans_r2c<8>(ctx, s, H, L1 * L2 * L3, L1, &done, L3);
      if (rc) return rc;
      if (!done) return fail(ctx, SRTB_B200_E_UNSUPPORTED, "r2c: four-sweep plan needs the TMA last sweep");
      return 0;
    }
    int l1, l2, l3 = 0;
    if (q <= 20) {
      l1 = (q + 1) / 2;
      l2 = q - l1;
    } else {
      plan3(q, &l1, &l2, &l3);
    }
    const int llast = l3 ? l3 : l2;
    if (llast >= 6 && llast <= 8 && get_encode_tiled()) {
      if (int rc = grow(ctx, ctx->lane.fft_scratch, M * sizeof(float2))) return rc;
      float2* s = ctx->lane.fft_scratch.p;
      const size_t L1 = (size_t)1 << l1, L2 = (size_t)1 << l2, L3 = (size_t)1 << l3;
      bool first_done = false;
      if (raw && raw->base) {
        // unpack fused into the first pass: the float buffer is not even written by an unpack kernel
        if (int rc = dispatch_col_raw(ctx, l1, *raw, s, l3 ? L2 * L3 : L2, &first_done)) return rc;
        if (raw_used) *raw_used = first_done;
        if (!first_done) return SRTB_B200_E_UNSUPPORTED;  // caller unpacks and retries without `raw`
      }
      if (!first_done)
        if (int rc = dispatch_col<true>(ctx, l1, H, s, 1, l3 ? L2 * L3 : L2)) return rc;
      if (l3)
        if (int rc = dispatch_col<true>(ctx, l2, s, s, L1, L3)) return rc;
      const size_t A = l3 ? L1 * L2 : L1;
      bool done = false;
      int rc = 0;
      switch (llast) {
        case 6: rc = launch_trans_r2c<6>(ctx, s, H, A, L1, &done); break;
        case 7: rc = launch_trans_r2c<7>(ctx, s, H, A, L1, &done); break;
        default: rc = launch_trans_r2c<8>(ctx, s, H, A, L1, &done); break;
      }
      if (rc) return rc;
      if (done) return 0;
      // tensor map refused: finish with the plain last pass + split kernel
      if (int rc2 = dispatch_trans<true>(ctx, llast, s, H, 1, A, L1)) return rc2;
      const unsigned grid = std::min<unsigned>(grid_for(ctx, M / 2 + 1, 256), 4096);
      CK(launch(ctx, false, r2c_post_kernel<true>, grid, 256, 0, H, M, ctx->lane.partial, ctx->lane.ticket, ctx->lane.mean));
      return 0;
    }
  }
  if (raw && raw->base) return SRTB_B200_E_UNSUPPORTED;  // fused unpack needs the multi-pass TMA route
  if (int rc = fft_c2c_impl<true>(ctx, H, M, 1)) return rc;
  const unsigned grid = std::min<unsigned>(grid_for(ctx, M / 2 + 1, 256), 4096);
  CK(launch(ctx, false, r2c_post_kernel<true>, grid, 256, 0, H, M, ctx->lane.partial, ctx->lane.ticket, ctx->lane.mean));
  return 0;
}

// ------------------------------------------------------------------------------------
// RFI stage 1
// ------------------------------------------------------------------------------------
extern "C" float srtb_b200_norm_coefficient(size_t in_count, size_t spectrum_channel_count) {
  // std::pow(float(Nc) * float(Nc) / float(C), -0.5) evaluated in double, stored as float
  return static_cast<float>(std::pow(
      static_cast<float>(in_count) * static_cast<float>(in_count) / static_cast<float>(spectrum_channel_count),
      -0.5));
}

// boost::split(..., token_compress_on): adjacent separators merge into one
static std::vector<std::string> split_compress(const std::string& s, char sep) {
  std::vector<std::string> out(1);
  bool prev_sep = false;
  for (char c : s) {
    if (c == sep) {
      if (!prev_sep) out.emplace_back();
      prev_sep = true;
    } else {
      out.back().push_back(c);
      prev_sep = false;
    }
  }
  return out;
}

extern "C" size_t srtb_b200_eval_rfi_ranges(const char* freq_list, float* pairs, size_t max_pairs) {
  // "a-b, c-d" (MHz): split on ',' then on '-'; entries that are not exactly two numbers are
  // skipped (the reference logs a warning, rfi_mitigation.hpp:76-78)
  if (!freq_list) return 0;
  size_t n = 0;
  for (const std::string& range : split_compress(freq_list, ',')) {
    const std::vector<std::string> nums = split_compress(range, '-');
    if (nums.size() != 2) continue;
    char* end = nullptr;
    const double f1 = std::strtod(nums[0].c_str(), &end);
    if (end == nums[0].c_str()) continue;
    const double f2 = std::strtod(nums[1].c_str(), &end);
    if (end == nums[1].c_str()) continue;
    if (pairs && n < max_pairs) {
      pairs[2 * n] = static_cast<float>(f1);
      pairs[2 * n + 1] = static_cast<float>(f2);
    }
    n++;
  }
  return n;
}

extern "C" int srtb_b200_rfi_range_to_bins(float f1, float f2, float freq_low, float bandwidth,
                                           size_t in_count, size_t* lo, size_t* hi) {
  if (std::signbit(bandwidth) != std::signbit(f2 - f1)) std::swap(f1, f2);
  const float scale = static_cast<float>(in_count - 1);
  const float a = std::round((f1 - freq_low) / bandwidth * scale);
  const float b = std::round((f2 - freq_low) / bandwidth * scale);
  if (!(a >= 0.0f) || !(b >= 0.0f) || a >= 1.8446744e19f || b >= 1.8446744e19f) return 0;
  const size_t l = static_cast<size_t>(a), h = static_cast<size_t>(b);
  if (l <= h && h < in_count) {
    if (lo) *lo = l;
    if (hi) *hi = h;
    return 1;
  }
  return 0;
}

// mitigate_rfi_manual (rfi_mitigation.hpp:97-158): zero the listed bin ranges, 16 ranges per launch. logp != 0: x holds
// the spectrum channel-blocked (bin k1 + 2^logp k2 at (k2 >> 3) 2^logq + 8 k1 + (k2 & 7), r2c_sweep_order)
static int zero_bin_ranges(srtb_b200_ctx* ctx, float2* x, const std::vector<size_t>& bins, unsigned logp = 0,
                           unsigned logq = 0) {
  for (size_t r0 = 0; r0 < bins.size() / 2; r0 += 16) {
    bin_ranges br;
    br.logp = logp;
    br.logq = logq;
    const size_t nr = std::min<size_t>(16, bins.size() / 2 - r0);
    size_t longest = 1;
    for (size_t r = 0; r < nr; r++) {
      br.lo[r] = bins[2 * (r0 + r)];
      br.hi[r] = bins[2 * (r0 + r) + 1];
      longest = std::max<size_t>(longest, br.hi[r] - br.lo[r] + 1);
    }
    dim3 g(grid_for(ctx, longest, 256), (unsigned)nr);
    CK(launch(ctx, true, rfi_zero_ranges_kernel, g, 256, 0, x, br));
  }
  return 0;
}

extern "C" int srtb_b200_rfi_s1(srtb_b200_ctx* ctx, void* d_x, size_t count, float avg_threshold,
                                float norm_coef, const size_t* h_bin_ranges, size_t n_ranges,
                                float* d_mean_out) {
  API_LOCK(ctx);
  if (!ctx || !d_x) return fail(ctx, SRTB_B200_E_INVALID, "rfi_s1: null argument");
  if (!aligned8(d_x)) return fail(ctx, SRTB_B200_E_INVALID, "rfi_s1: d_x is not 8-byte aligned");
  if (count == 0) return fail(ctx, SRTB_B200_E_INVALID, "rfi_s1: zero count");
  if (n_ranges && !h_bin_ranges) return fail(ctx, SRTB_B200_E_INVALID, "rfi_s1: null ranges");
  const std::vector<size_t> bins(h_bin_ranges, h_bin_ranges + 2 * n_ranges);
  for (size_t r = 0; r < n_ranges; r++)
    if (!(bins[2 * r] <= bins[2 * r + 1] && bins[2 * r + 1] < count))
      return fail(ctx, SRTB_B200_E_INVALID, "rfi_s1: bin range out of bounds");
  CK(cudaSetDevice(ctx->device));
  stage_scope stats_(ctx, SRTB_B200_STAGE_RFI_S1, 24.0 * (double)count);
  float2* x = static_cast<float2*>(d_x);
  const unsigned grid = std::min<unsigned>(grid_for(ctx, count / 2 + 1, 256), 4096);
  CK(launch(ctx, false, power_sum_kernel, grid, 256, 0, x, count, ctx->lane.partial, ctx->lane.ticket, ctx->lane.mean));
  if (d_mean_out) CK(cudaMemcpyAsync(d_mean_out, ctx->lane.mean, sizeof(float), cudaMemcpyDeviceToDevice, ctx->lane.stream));
  CK(launch(ctx, false, rfi_s1_apply_kernel, grid_for(ctx, count / 2 + 1, 256), 256, 0, x, count, ctx->lane.mean,
            avg_threshold, norm_coef));
  return zero_bin_ranges(ctx, x, bins);
}

// ------------------------------------------------------------------------------------
// dedisperse
// ------------------------------------------------------------------------------------
extern "C" int srtb_b200_dedisperse(srtb_b200_ctx* ctx, void* d_x, size_t count, float f_min, float f_c,
                                    float df, float dm) {
  API_LOCK(ctx);
  if (!ctx || !d_x) return fail(ctx, SRTB_B200_E_INVALID, "dedisperse: null argument");
  if (!aligned8(d_x)) return fail(ctx, SRTB_B200_E_INVALID, "dedisperse: d_x is not 8-byte aligned");
  if (count == 0) return 0;
  CK(cudaSetDevice(ctx->device));
  stage_scope stats_(ctx, SRTB_B200_STAGE_DEDISPERSE, 16.0 * (double)count);
  constexpr double D = 4.148808e3;  // coherent_dedispersion.hpp:67
  const double ddm = (D * 1e6) * (double)dm;
  CK(launch(ctx, false, dedisperse_kernel<false>, grid_for(ctx, count / 2 + 1, 256, 16), 256, 0,
            static_cast<const float2*>(d_x), static_cast<float2*>(d_x), count, (double)f_min, (double)df, (double)f_c, ddm,
            nullptr, 0.f, 1.f));
  return 0;
}

// s1 (mean -> zap/normalise) and the chirp in two kernels instead of three: power sum, then one
// fused apply + chirp sweep, then the manual zap (zero * chirp = zero, so the order is equivalent). The mean is
// already in the lane's `mean` (left there by the R2C); src is the spectrum read, x the one written (may be equal).
static int rfi_s1_dedisperse_fused(srtb_b200_ctx* ctx, float2* x, const float2* src, size_t count, float avg_threshold,
                                   float coef, const std::vector<size_t>& bins, float f_min, float f_c, float df, float dm) {
  constexpr double D = 4.148808e3;
  const double ddm = (D * 1e6) * (double)dm;
  CK(launch(ctx, false, dedisperse_kernel<true>, grid_for(ctx, count / 2 + 1, 256, 16), 256, 0, src, x, count,
            (double)f_min, (double)df, (double)f_c, ddm, ctx->lane.mean, avg_threshold, coef));
  return zero_bin_ranges(ctx, x, bins);
}

extern "C" size_t srtb_b200_nsamps_reserved(size_t baseband_input_count, size_t spectrum_channel_count,
                                            float freq_low, float bandwidth, float sample_rate, float dm,
                                            int reserve_sample) {
  if (!reserve_sample) return 0;
  constexpr double D = 4.148808e3;
  const float f = freq_low + bandwidth, f_c = freq_low;
  const float delay = static_cast<float>(-D * (double)dm * (1.0 / (double)(f * f) - 1.0 / (double)(f_c * f_c)));
  const float minimal_f = 2 * std::round(delay * sample_rate);
  const size_t minimal = static_cast<size_t>(minimal_f < 0 ? 0.0f : minimal_f);
  const size_t per_bin = spectrum_channel_count * 2;
  const long long keep = static_cast<long long>(baseband_input_count - minimal) / (long long)per_bin * (long long)per_bin;
  if (keep > 0) return baseband_input_count - (size_t)keep;
  return 0;
}

// ------------------------------------------------------------------------------------
// RFI stage 2 (spectral kurtosis)
// ------------------------------------------------------------------------------------
// a channel is kept when its SK estimate over M time samples lies in [lo, hi]
struct sk_range {
  float lo, hi;
};
static sk_range sk_bounds(float sk_threshold, size_t M) {
  const float M_ = static_cast<float>(M);
  float hi = sk_threshold, lo = 2 - sk_threshold;
  if (lo > hi) std::swap(lo, hi);
  return {lo * ((M_ - 1) / (M_ + 1)) + 1, hi * ((M_ - 1) / (M_ + 1)) + 1};
}

extern "C" int srtb_b200_rfi_s2_sk(srtb_b200_ctx* ctx, void* d_x, size_t time_count, size_t chan_count,
                                   float sk_threshold, float* d_sk_out) {
  API_LOCK(ctx);
  if (!ctx || !d_x) return fail(ctx, SRTB_B200_E_INVALID, "rfi_s2: null argument");
  if (!aligned8(d_x)) return fail(ctx, SRTB_B200_E_INVALID, "rfi_s2: d_x is not 8-byte aligned");
  if (time_count == 0 || chan_count == 0) return fail(ctx, SRTB_B200_E_INVALID, "rfi_s2: zero size");
  CK(cudaSetDevice(ctx->device));
  stage_scope stats_(ctx, SRTB_B200_STAGE_RFI_S2, 8.0 * (double)time_count * (double)chan_count);
  const auto [lo_, hi_] = sk_bounds(sk_threshold, time_count);
  CK(launch(ctx, false, sk_kernel, (unsigned)chan_count, 256, 0, static_cast<float2*>(d_x), time_count, lo_, hi_, d_sk_out));
  return 0;
}

// ------------------------------------------------------------------------------------
// signal detect
// ------------------------------------------------------------------------------------
// where one detector run writes: the series, result header d_res[slot] and sample count of the context's `slot`, and,
// each already offset to this run by the caller (or null), the pinned host rows [MAX_BOXCARS][L] of its positive
// series, its raw column sums [L] and its peak record. header_zeroed: the caller zeroed d_res[slot] before the first
// kernel (a memset between two kernels would break their programmatic-dependent-launch chain).
struct detect_out {
  int slot = 0;
  float* host_series = nullptr;
  float* raw = nullptr;
  detect_dev_peak* peak = nullptr;
  bool header_zeroed = false;
};

// time samples of a row of time_count the detector searches: the reserved tail is left out unless it is the whole row
static size_t detected_samples(size_t time_count, size_t reserved) {
  return time_count <= reserved ? time_count : time_count - reserved;
}

// boxcar kernel CTAs for a series of ts samples: one per possible boxcar; those beyond n_boxcars (known only on the
// device) exit at once
static unsigned boxcar_ctas(size_t max_boxcar, size_t ts) {
  unsigned n = 1;
  for (size_t b = 2; b <= max_boxcar && b < ts && n < SRTB_B200_MAX_BOXCARS; b *= 2) n++;
  return n;
}

static int detect_prepare(srtb_b200_ctx* ctx, int slot, size_t time_count, size_t need_partial_elems) {
  if (int rc = grow(ctx, ctx->series[slot], (size_t)SRTB_B200_MAX_BOXCARS * time_count * sizeof(float))) return rc;
  if (int rc = grow(ctx, ctx->lane.acc, time_count * sizeof(float))) return rc;
  return grow(ctx, ctx->lane.colsum_partial, need_partial_elems * sizeof(float));
}

// channel rows in chunks for colsum_partial_kernel: about 8 CTAs per SM in all, at most 128 chunks
struct colsum_chunks {
  size_t ctas_per_chunk, rows_per_chunk, chunks;
};
static colsum_chunks colsum_geometry(const srtb_b200_ctx* ctx, size_t samples_per_row, size_t chan_count) {
  const size_t ctas_per_chunk = (samples_per_row + 511) / 512;
  size_t chunks = std::max<size_t>(1, (size_t)ctx->sm_count * 8 / ctas_per_chunk);
  chunks = std::min(chunks, std::min<size_t>(128, chan_count));
  const size_t rows_per_chunk = (chan_count + chunks - 1) / chunks;
  return {ctas_per_chunk, rows_per_chunk, (chan_count + rows_per_chunk - 1) / rows_per_chunk};
}

// column-sum reduction over `chunks` partial rows, zero count, scan, boxcar ladder
// partial: the `chunks` rows of partial column sums, or null when out.slot's series already holds the summed series
// (the total-intensity sum, whose tail is not a stage of its own and so is not timed)
// zero_stride / zero_count_n: where the detector looks for masked channels — the first time sample of every channel
// of [C][L] (stride L, C of them; the default), or the first spectrum of [time][frequency] (stride 1; v1 detector, and
// the sum's channel mask)
static int detect_tail(srtb_b200_ctx* ctx, const detect_out& out, const float* partial, const float2* x,
                       size_t time_count, size_t chan_count, size_t ts_count, size_t chunks, float snr, float chan_thr,
                       size_t max_boxcar, size_t zero_stride = 0) {
  if (zero_stride == 0) zero_stride = time_count;
  const int slot = out.slot;
  std::optional<stage_scope> stats_;
  if (partial) stats_.emplace(ctx, SRTB_B200_STAGE_FUSED_DETECT_TAIL, 4.0 * (double)chunks * (double)ts_count);
  const size_t scan_ctas = partial ? (ts_count + 31) / 32 : (chan_count + 1023) / 1024;
  CK(launch(ctx, true, colsum_final_scan_kernel, (unsigned)std::min<size_t>(scan_ctas, (size_t)ctx->sm_count), 1024, 0,
            partial, ts_count, chunks, ctx->series[slot].p, ctx->lane.acc.p, x, zero_stride, chan_count, chan_thr,
            max_boxcar, ctx->lane.detect_ticket, ctx->d_res + slot, (size_t)0, (size_t)0, out.raw));
  auto boxcar = out.peak ? detect_boxcar_kernel<true> : detect_boxcar_kernel<false>;
  CK(launch(ctx, true, boxcar, boxcar_ctas(max_boxcar, ts_count), 1024, 0, ctx->series[slot].p, time_count,
            (const float*)ctx->lane.acc.p, ts_count, snr, ctx->d_res + slot, out.host_series, out.peak, (size_t)0,
            (size_t)0));
  ctx->series_len[slot] = time_count;
  return 0;
}

static int detect_enqueue(srtb_b200_ctx* ctx, const detect_out& out, const float2* x, size_t time_count,
                          size_t chan_count, size_t time_reserved_count, float snr, float chan_thr,
                          size_t max_boxcar) {
  const size_t ts_count = detected_samples(time_count, time_reserved_count);
  const colsum_chunks cg = colsum_geometry(ctx, ts_count, chan_count);
  if (int rc = detect_prepare(ctx, out.slot, time_count, cg.chunks * ts_count)) return rc;
  CK(cudaMemsetAsync(ctx->d_res + out.slot, 0, sizeof(detect_dev_result), ctx->lane.stream));
  dim3 g((unsigned)cg.ctas_per_chunk, (unsigned)cg.chunks);
  CK(launch(ctx, false, colsum_partial_kernel, g, 256, 0, const_cast<float2*>(x), time_count, chan_count, ts_count,
            cg.rows_per_chunk, ctx->lane.colsum_partial.p, nullptr));
  return detect_tail(ctx, out, ctx->lane.colsum_partial.p, x, time_count, chan_count, ts_count, cg.chunks, snr, chan_thr,
                     max_boxcar);
}

// watfft (backward C2C of every channel row) with spectral kurtosis + the detector's partial column
// sums fused into its epilogue: the dynamic spectrum is written once and not read again until the
// candidate sink. Used by process_block when one CTA holds a whole row (L = 512 .. 4096).
// s1 + chirp folded into the waterfall kernel's load: the sixteen-point row kernels (L = 1024..4096) and the
// whole-row kernel (L = 8192, 16384)
static bool chirp_fusable(size_t time_count) {
  return time_count == 1024 || time_count == 2048 || time_count == 4096 || time_count == 8192 || time_count == 16384;
}

template <int LOGL>
static int watfft_sk_launch(srtb_b200_ctx* ctx, float2* x, size_t chan_count, float lo_, float hi_, size_t ts_count,
                            size_t* chunks_out, const row_chirp_params* chirp = nullptr, const float2* src = nullptr) {
  if (!src) src = x;  // in place unless the input spectrum is kept (DM sweep)
  unsigned grid = 1;
  const float2* tw = nullptr;
  if constexpr (LOGL >= 10) {  // sixteen-point row kernel; L = 512 has the eight-point one only
    constexpr int T16 = row16_t<LOGL>::value, threads = ((1 << LOGL) / 16) * T16;
    // block buffers are 16-byte aligned, so rows of these lengths always take the chirp-on-load route
    if (!chirp) return fail(ctx, SRTB_B200_E_UNSUPPORTED, "watfft: the sixteen-point SK row kernel needs the fused chirp");
    auto kern = fft_row16_tma_kernel<LOGL, T16, false, true, true>;
    constexpr size_t smem = row16_smem<LOGL, T16>::bytes;
    const size_t ntiles = (chan_count + T16 - 1) / T16;
    if (int rc = persistent_grid(ctx, kern, threads, smem, smem, ntiles, &grid)) return rc;
    if (int rc = grow(ctx, ctx->lane.colsum_partial, (size_t)grid * ts_count * sizeof(float))) return rc;
    if (int rc = get_stage_twiddles(ctx, LOGL, &tw)) return rc;
    row_sk_params p{lo_, hi_, ctx->lane.colsum_partial.p, (unsigned)ts_count};
    CK(launch(ctx, true, kern, grid, threads, smem, src, x, chan_count, tw, p, chirp ? *chirp : row_chirp_params{}));
  } else {
    if (chirp || src != x) return fail(ctx, SRTB_B200_E_UNSUPPORTED, "watfft: fused chirp needs the sixteen-point row kernel");
    constexpr int T = row_t<LOGL>::value;
    auto kern = fft_row_tma_kernel<LOGL, T, false, true>;
    constexpr size_t smem = row_tma_smem<LOGL, T>::bytes;
    const size_t ntiles = (chan_count + T - 1) / T;
    if (int rc = persistent_grid(ctx, kern, pass_threads<LOGL, T>::value, smem, smem, ntiles, &grid)) return rc;
    if (int rc = grow(ctx, ctx->lane.colsum_partial, (size_t)grid * ts_count * sizeof(float))) return rc;
    if (int rc = get_stage_twiddles(ctx, LOGL, &tw)) return rc;
    row_sk_params p{lo_, hi_, ctx->lane.colsum_partial.p, (unsigned)ts_count};
    CK(launch(ctx, false, kern, grid, pass_threads<LOGL, T>::value, smem, x, x, chan_count, tw, p));
  }
  *chunks_out = grid;
  return 0;
}

static int watfft_sk_detect_fused(srtb_b200_ctx* ctx, const detect_out& out, float2* x, size_t time_count, size_t chan_count,
                                  size_t time_reserved_count, float sk_threshold, float snr, float chan_thr,
                                  size_t max_boxcar, const row_chirp_params* chirp = nullptr,
                                  const float2* src = nullptr, bool sweep_order = false) {
  const size_t ts_count = detected_samples(time_count, time_reserved_count);
  if (int rc = detect_prepare(ctx, out.slot, time_count, 1)) return rc;
  if (!out.header_zeroed) CK(cudaMemsetAsync(ctx->d_res + out.slot, 0, sizeof(detect_dev_result), ctx->lane.stream));
  const auto [lo_, hi_] = sk_bounds(sk_threshold, time_count);
  size_t chunks = 0;
  int rc = 0;
  std::unique_ptr<stage_scope> stats_(new stage_scope(ctx, SRTB_B200_STAGE_FUSED_WATERFALL, 16.0 * (double)time_count * (double)chan_count));
  if (time_count == 8192 || time_count == 16384) {
    row_sk_params p{lo_, hi_, nullptr, (unsigned)ts_count};
    row_chirp_params cpv{};
    if (chirp) {
      cpv = *chirp;
      // 1/f of a bin comes from Newton steps off the reciprocal of the bin B1 = L/16 below; n steps leave a relative
      // error of (B1 df / f)^(2^n). One step when that is within an ulp of fp64 (2^-52: as good as the division the
      // reference performs; the J1644 shape has 1.5e-16), two when the fourth power keeps |k| * error below 1e-9
      // cycles of phase, else the exact reciprocal of every bin (widely spaced bins of short test blocks).
      const double fa = std::min(std::fabs(cpv.f_min), std::fabs(cpv.f_c));
      const double delta = (double)(time_count / 16) * std::fabs(cpv.df) / fa;
      const double q = (cpv.f_c - cpv.f_min) * cpv.inv_fc;
      const double kmax = std::max(1.0, std::fabs(cpv.ddm) / fa * q * q);
      // two distances: B1 bins (along a butterfly's inputs) and 1 bin (the pair's second column)
      const double d2 = delta * delta;
      const double dn = std::fabs(cpv.df) / fa, dn2 = dn * dn;
      const int far_steps = (d2 <= 0x1p-52) ? 1 : ((d2 * d2 * kmax < 1e-9) ? 2 : 0);
      const int near_steps = (dn2 <= 0x1p-52) ? 1 : ((dn2 * dn2 * kmax < 1e-9) ? 2 : 0);
      // kernel variants: 1 = (1, 1), 3 = (2, 1), 4 = (2, 2), 2 = exact
      cpv.newton = (far_steps == 0 || near_steps == 0) ? 2
                   : (far_steps == 1 ? 1 : (near_steps == 1 ? 3 : 4));
      if (cpv.phase) cpv.newton = 5;  // tabulated phases (block path): no reciprocal at all
      if (sweep_order) cpv.newton = 2;  // every bin's phase evaluated exactly as the table would hold it
    }
    const float2* s_ = src ? src : x;
    rc = (time_count == 8192) ? launch_bigrow<13, false>(ctx, s_, x, chan_count, &p, chirp ? &cpv : nullptr, &chunks)
                              : launch_bigrow<14, false>(ctx, s_, x, chan_count, &p, chirp ? &cpv : nullptr, &chunks,
                                                         sweep_order);
    if (rc) return rc;
    stats_.reset();
    return detect_tail(ctx, out, ctx->lane.colsum_partial.p, x, time_count, chan_count, ts_count, chunks, snr, chan_thr,
                       max_boxcar);
  }
  switch (ilog2(time_count)) {
    case 9: rc = watfft_sk_launch<9>(ctx, x, chan_count, lo_, hi_, ts_count, &chunks, chirp, src); break;
    case 10: rc = watfft_sk_launch<10>(ctx, x, chan_count, lo_, hi_, ts_count, &chunks, chirp, src); break;
    case 11: rc = watfft_sk_launch<11>(ctx, x, chan_count, lo_, hi_, ts_count, &chunks, chirp, src); break;
    default: rc = watfft_sk_launch<12>(ctx, x, chan_count, lo_, hi_, ts_count, &chunks, chirp, src); break;
  }
  if (rc) return rc;
  stats_.reset();
  return detect_tail(ctx, out, ctx->lane.colsum_partial.p, x, time_count, chan_count, ts_count, chunks, snr, chan_thr,
                     max_boxcar);
}

// Rows longer than one CTA's shared memory (2^15 .. 2^20 time samples; the shipped configurations have 2^18):
//   sweep A  column FFTs with rfi_mitigation_s1 + the chirp applied as the tile is read  (spectrum -> scratch)
//   sweep B  transposing last sweep, leaving per-tile (sum |y|^2, sum |y|^4)              (scratch -> spectrum)
//   decide   one thread per channel folds its tiles and takes the SK decision
//   sums     the detector's partial column sums, zeroing the flagged rows on the way (one read of the spectrum)
// i.e. 20 bytes per sample instead of the 32 of dedisperse + two-sweep waterfall + SK + column sums.
// (16-byte aligned spectra only)
static bool long_fusable(size_t time_count) {
  const int q = ilog2(time_count);
  return is_pow2(time_count) && q >= 15 && q <= 18 && get_encode_tiled();
}

static int watfft_long_fused(srtb_b200_ctx* ctx, const detect_out& out, float2* x, const float2* src, size_t time_count,
                             size_t chan_count, size_t time_reserved_count, float sk_threshold, float snr,
                             float chan_thr, size_t max_boxcar, const row_chirp_params& chirp) {
  const size_t ts_count = detected_samples(time_count, time_reserved_count);
  const int q = ilog2(time_count);
  const int l1 = (q + 1) / 2, l2 = q - l1;
  const size_t L1 = (size_t)1 << l1, L2 = (size_t)1 << l2;
  if (int rc = grow(ctx, ctx->lane.fft_scratch, chan_count * time_count * sizeof(float2))) return rc;
  float2* s = ctx->lane.fft_scratch.p;
  const size_t T_last = (l2 <= 8) ? 16 : 8;  // rows per tile of the last sweep (col_t)
  const size_t tiles_per_row = L1 / T_last;
  if (int rc = grow(ctx, ctx->lane.long_stats, chan_count * tiles_per_row * sizeof(float2))) return rc;
  if (int rc = grow(ctx, ctx->lane.long_zap, chan_count)) return rc;
  float2* stats = ctx->lane.long_stats.p;
  unsigned char* zap = ctx->lane.long_zap.p;
  row_chirp_params cp = chirp;
  {
    // Newton steps for 1/f between a thread's consecutive points, U * B = (L1 / 16) * L2 bins apart
    const double fa = std::min(std::fabs(cp.f_min), std::fabs(cp.f_c));
    const double delta = (double)((L1 / 16) * L2) * std::fabs(cp.df) / fa, d2 = delta * delta;
    const double qq = (cp.f_c - cp.f_min) * cp.inv_fc;
    const double kmax = std::max(1.0, std::fabs(cp.ddm) / fa * qq * qq);
    cp.newton = (d2 <= 0x1p-52) ? 1 : ((d2 * d2 * kmax < 1e-9) ? 2 : 0);
  }
  std::unique_ptr<stage_scope> stats_(new stage_scope(ctx, SRTB_B200_STAGE_FUSED_WATERFALL, 40.0 * (double)time_count * (double)chan_count));
  bool done = false;
  int rc = 0;
  switch (l1) {
    case 8: rc = launch_col_tma<8, false>(ctx, src, s, chan_count, L2, &done, &cp); break;
    case 9: rc = launch_col_tma<9, false>(ctx, src, s, chan_count, L2, &done, &cp); break;
    default: break;
  }
  if (rc) return rc;
  if (!done) return SRTB_B200_E_UNSUPPORTED;
  done = false;
  switch (l2) {
    case 7: rc = launch_trans_tma<7, false>(ctx, s, x, chan_count, L1, L1, &done, 0, stats); break;
    case 8: rc = launch_trans_tma<8, false>(ctx, s, x, chan_count, L1, L1, &done, 0, stats); break;
    case 9: rc = launch_trans_tma<9, false>(ctx, s, x, chan_count, L1, L1, &done, 0, stats); break;
    default: break;
  }
  if (rc) return rc;
  if (!done) return fail(ctx, SRTB_B200_E_UNSUPPORTED, "watfft: long fused plan needs the TMA last sweep");
  const auto [lo_, hi_] = sk_bounds(sk_threshold, time_count);
  CK(launch(ctx, false, sk_decide_kernel, (unsigned)((chan_count + 255) / 256), 256, 0, stats, (unsigned)tiles_per_row,
            chan_count, static_cast<float>(time_count), lo_, hi_, zap));
  // partial column sums (all time samples are visited so that flagged rows are zeroed completely)
  const colsum_chunks cg = colsum_geometry(ctx, time_count, chan_count);
  if (int rc2 = detect_prepare(ctx, out.slot, time_count, cg.chunks * ts_count)) return rc2;
  if (!out.header_zeroed) CK(cudaMemsetAsync(ctx->d_res + out.slot, 0, sizeof(detect_dev_result), ctx->lane.stream));
  dim3 g((unsigned)cg.ctas_per_chunk, (unsigned)cg.chunks);
  CK(launch(ctx, false, colsum_partial_kernel, g, 256, 0, x, time_count, chan_count, ts_count, cg.rows_per_chunk,
            ctx->lane.colsum_partial.p, zap));
  stats_.reset();
  return detect_tail(ctx, out, ctx->lane.colsum_partial.p, x, time_count, chan_count, ts_count, cg.chunks, snr, chan_thr,
                     max_boxcar);
}

static int detect_collect(srtb_b200_ctx* ctx, int slot, srtb_b200_detect_result* h_result, float* h_series,
                          int copy_all) {
  std::memcpy(h_result, ctx->h_res + slot, sizeof(srtb_b200_detect_result));
  if (h_series && h_result->detect_enabled) {
    const size_t stride = ctx->series_len[slot];
    bool any = false;
    for (int b = 0; b < h_result->n_boxcars; b++) {
      if (copy_all || h_result->signal_count[b] > 0) {
        CK(cudaMemcpyAsync(h_series + (size_t)b * stride, ctx->series[slot].p + (size_t)b * stride,
                           h_result->series_length[b] * sizeof(float), cudaMemcpyDeviceToHost, ctx->lane.stream));
        any = true;
      }
    }
    if (any) CK(cudaStreamSynchronize(ctx->lane.stream));
  } else if (h_series && copy_all) {
    // detection disabled: still hand back the mean-removed time series
    CK(cudaMemcpyAsync(h_series, ctx->series[slot].p, h_result->time_series_count * sizeof(float),
                       cudaMemcpyDeviceToHost, ctx->lane.stream));
    CK(cudaStreamSynchronize(ctx->lane.stream));
  }
  return 0;
}

extern "C" int srtb_b200_signal_detect(srtb_b200_ctx* ctx, const void* d_x, size_t time_count,
                                       size_t chan_count, size_t time_reserved_count, float snr_threshold,
                                       float channel_threshold, size_t max_boxcar_length,
                                       srtb_b200_detect_result* h_result, float* h_series, int copy_all) {
  API_LOCK(ctx);
  if (!ctx || !d_x || !h_result) return fail(ctx, SRTB_B200_E_INVALID, "signal_detect: null argument");
  if (!aligned8(d_x)) return fail(ctx, SRTB_B200_E_INVALID, "signal_detect: d_x is not 8-byte aligned");
  if (time_count == 0 || chan_count == 0) return fail(ctx, SRTB_B200_E_INVALID, "signal_detect: zero size");
  CK(cudaSetDevice(ctx->device));
  stage_scope stats_(ctx, SRTB_B200_STAGE_SIGNAL_DETECT, 8.0 * (double)time_count * (double)chan_count);
  if (int rc = detect_enqueue(ctx, detect_out{}, static_cast<const float2*>(d_x), time_count, chan_count,
                              time_reserved_count, snr_threshold, channel_threshold, max_boxcar_length))
    return rc;
  CK(cudaMemcpyAsync(ctx->h_res, ctx->d_res, sizeof(detect_dev_result), cudaMemcpyDeviceToHost, ctx->lane.stream));
  CK(cudaStreamSynchronize(ctx->lane.stream));
  return detect_collect(ctx, 0, h_result, h_series, copy_all);
}

// ---- alternates of the refft path: spectra laid out [time][frequency] ------------------------------------------
static int sk_v1_enqueue(srtb_b200_ctx* ctx, float2* x, size_t fft_bins, size_t time_counts, float sk_threshold,
                         float* d_sk_out) {
  if (int rc = grow(ctx, ctx->lane.long_zap, fft_bins)) return rc;
  unsigned char* zap = ctx->lane.long_zap.p;
  const auto [lo_, hi_] = sk_bounds(sk_threshold, time_counts);
  CK(launch(ctx, false, sk_v1_stats_kernel, (unsigned)((fft_bins + 31) / 32), 256, 0, x, fft_bins, time_counts, lo_, hi_,
            zap, d_sk_out));
  const unsigned gy = (unsigned)std::max<size_t>(1, std::min<size_t>(time_counts, 64));
  CK(launch(ctx, false, sk_v1_zero_kernel, dim3((unsigned)((fft_bins + 255) / 256), gy), 256, 0, x, fft_bins, time_counts,
            zap));
  return 0;
}

extern "C" int srtb_b200_rfi_sk_v1(srtb_b200_ctx* ctx, void* d_x, size_t fft_bins, size_t time_counts,
                                   float sk_threshold, float* d_sk_out) {
  API_LOCK(ctx);
  if (!ctx || !d_x) return fail(ctx, SRTB_B200_E_INVALID, "rfi_sk_v1: null argument");
  if (!aligned8(d_x)) return fail(ctx, SRTB_B200_E_INVALID, "rfi_sk_v1: d_x is not 8-byte aligned");
  if (fft_bins == 0 || time_counts == 0) return fail(ctx, SRTB_B200_E_INVALID, "rfi_sk_v1: zero size");
  CK(cudaSetDevice(ctx->device));
  return sk_v1_enqueue(ctx, static_cast<float2*>(d_x), fft_bins, time_counts, sk_threshold, d_sk_out);
}

extern "C" int srtb_b200_signal_detect_v1(srtb_b200_ctx* ctx, void* d_x, size_t count_per_batch, size_t batch_size,
                                          float sk_threshold, float snr_threshold, float channel_threshold,
                                          size_t max_boxcar_length, srtb_b200_detect_result* h_result, float* h_series,
                                          int copy_all) {
  API_LOCK(ctx);
  if (!ctx || !d_x || !h_result) return fail(ctx, SRTB_B200_E_INVALID, "signal_detect_v1: null argument");
  if (!aligned8(d_x)) return fail(ctx, SRTB_B200_E_INVALID, "signal_detect_v1: d_x is not 8-byte aligned");
  if (count_per_batch == 0 || batch_size == 0) return fail(ctx, SRTB_B200_E_INVALID, "signal_detect_v1: zero size");
  CK(cudaSetDevice(ctx->device));
  float2* x = static_cast<float2*>(d_x);
  if (int rc = sk_v1_enqueue(ctx, x, count_per_batch, batch_size, sk_threshold, nullptr)) return rc;
  // one value per spectrum; then the same tail as the v2 detector (mean removal, scan, boxcars) on a series of
  // batch_size values, masked channels counted over the first spectrum
  if (int rc = detect_prepare(ctx, 0, batch_size, batch_size)) return rc;
  CK(cudaMemsetAsync(ctx->d_res, 0, sizeof(detect_dev_result), ctx->lane.stream));
  CK(launch(ctx, false, rowsum_norm_kernel, (unsigned)((batch_size + 7) / 8), 256, 0, x, count_per_batch, batch_size,
            ctx->lane.colsum_partial.p));
  if (int rc = detect_tail(ctx, detect_out{}, ctx->lane.colsum_partial.p, x, batch_size, count_per_batch, batch_size, 1,
                           snr_threshold, channel_threshold, max_boxcar_length, /*zero_stride=*/1))
    return rc;
  CK(cudaMemcpyAsync(ctx->h_res, ctx->d_res, sizeof(detect_dev_result), cudaMemcpyDeviceToHost, ctx->lane.stream));
  CK(cudaStreamSynchronize(ctx->lane.stream));
  return detect_collect(ctx, 0, h_result, h_series, copy_all);
}

// ------------------------------------------------------------------------------------
// whole block
// ------------------------------------------------------------------------------------
static int format_streams(int format) {
  switch (format) {
    case SRTB_B200_FORMAT_SIMPLE: return 1;
    case SRTB_B200_FORMAT_INTERLEAVED_2:
    case SRTB_B200_FORMAT_NAOCPSR_SNAP1:
    case SRTB_B200_FORMAT_GZNUPSR_A1_2: return 2;
    case SRTB_B200_FORMAT_GZNUPSR_A1_4: return 4;
    default: return 0;
  }
}

// unpack fused into the first FFT sweep: possible when the samples are 8-bit, the window is the rectangle and every
// complex point of a stream is one fixed-size byte group (simple, "1 1 2 2", "1 2 1 2"); fills raw[stream]
static bool raw_sources_for(const srtb_b200_block_config* cfg, const void* d_baseband, size_t baseband_bytes, int streams,
                            raw_source (&raw)[4]) {
  const int bits = cfg->baseband_input_bits;
  const int fmt = cfg->baseband_format;
  const size_t N = cfg->baseband_input_count;
  // SRTB_B200_NO_FUSED_UNPACK forces the unpack kernel: the test of the fused first sweep compares both routes with it
  if (cfg->window != SRTB_B200_WINDOW_RECTANGLE || N < ((size_t)1 << 14) || !get_encode_tiled() ||
      std::getenv("SRTB_B200_NO_FUSED_UNPACK"))
    return false;
  if ((bits == 2 || bits == 4) && fmt == SRTB_B200_FORMAT_SIMPLE && baseband_bytes * 8 >= N * (size_t)bits) {
    // packed unsigned samples (the shipped J1644 configuration is 2-bit): decoded in the first sweep's stage 0
    raw[0].base = d_baseband;
    raw[0].bits = bits;
    raw[0].is_signed = false;
    return true;
  }
  if (!((bits == 8 || bits == -8) && baseband_bytes >= N * (size_t)streams)) return false;
  if (!(fmt == SRTB_B200_FORMAT_SIMPLE || (fmt == SRTB_B200_FORMAT_NAOCPSR_SNAP1 && bits == -8) ||
        fmt == SRTB_B200_FORMAT_INTERLEAVED_2 || fmt == SRTB_B200_FORMAT_GZNUPSR_A1_2))
    return false;
  for (int s = 0; s < streams; s++) {
    raw[s].base = d_baseband;
    raw[s].is_signed = (bits < 0);
    raw[s].G = 2 * streams;
    if (fmt == SRTB_B200_FORMAT_SIMPLE) { raw[s].o0 = 0; raw[s].o1 = 1; }
    else if (fmt == SRTB_B200_FORMAT_NAOCPSR_SNAP1) { raw[s].o0 = 2 * s; raw[s].o1 = 2 * s + 1; }
    else if (fmt == SRTB_B200_FORMAT_GZNUPSR_A1_2) {
      // words of four int8 samples alternate between the two streams (unpack.hpp:338-369): point m of stream s is at
      // byte 4 m + 4 s - 2 (m & 1); always read as signed (the reference casts to int8 whatever the sign of `bits`)
      raw[s].o0 = 4 * s;
      raw[s].o1 = 4 * s + 1;
      raw[s].delta = 2;
      raw[s].is_signed = true;
    }
    else { raw[s].o0 = s; raw[s].o1 = s + 2; }
  }
  return true;
}

// K12 phase table for the whole-row waterfall kernel (natural-order block path; the sweep-order route, the DM sweep,
// and tables above 4 GiB, evaluate every phase on the fly). Rebuilt when the geometry or the DM changes; built
// synchronously, so both lanes and any later launch may read it.
static int get_chirp_table(srtb_b200_ctx* ctx, size_t n, const row_chirp_params& cp, const float** out) {
  *out = nullptr;
  if (n * sizeof(float) > ((size_t)4 << 30)) return 0;
  const double key[6] = {(double)n, cp.f_min, cp.df, cp.inv_fc, cp.f_c, cp.ddm};
  if (ctx->chirp_tab.p && std::memcmp(key, ctx->chirp_tab_key, sizeof(key)) == 0) {
    *out = ctx->chirp_tab.p;
    return 0;
  }
  if (int rc = grow(ctx, ctx->chirp_tab, n * sizeof(float))) return rc;
  if (int rc = sync_lanes(ctx)) return rc;  // a block still in flight may be reading the previous table
  // a synchronous table build, like the twiddle uploads: not counted as a launch
  chirp_phase_table_kernel<<<grid_for(ctx, n, 256), 256, 0, ctx->lane.stream>>>(ctx->chirp_tab.p, n, cp.f_min, cp.df, cp.inv_fc,
                                                                           cp.f_c, cp.ddm);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(ctx->lane.stream));
  std::memcpy(ctx->chirp_tab_key, key, sizeof(key));
  *out = ctx->chirp_tab.p;
  return 0;
}

// second lane of a context (see lane_state): created on first use
static int ensure_alt_lane(srtb_b200_ctx* ctx) {
  if (ctx->alt_ready) return 0;
  CK(cudaStreamCreateWithFlags(&ctx->alt.stream, cudaStreamNonBlocking));
  CK(lane_alloc(&ctx->alt));
  CK(cudaEventCreateWithFlags(&ctx->lane_fork, cudaEventDisableTiming));
  CK(cudaEventCreateWithFlags(&ctx->lane_join, cudaEventDisableTiming));
  ctx->alt_ready = true;
  return 0;
}

// called on the first lane: the second lane continues from this point of it
static int fork_lanes(srtb_b200_ctx* ctx) {
  CK(cudaEventRecord(ctx->lane_fork, ctx->lane.stream));
  CK(cudaStreamWaitEvent(ctx->alt.stream, ctx->lane_fork, 0));
  return 0;
}

// what a block's configuration fixes for every one of its data streams
struct block_params {
  const srtb_b200_block_config* cfg = nullptr;
  int streams = 0;
  size_t N = 0, Nc = 0, batch = 0, L = 0;  // samples per stream, spectrum bins, channel rows, time samples per row
  std::vector<size_t> bins;                // manual zap ranges as (lo, hi) bin pairs
  float coef = 0, f_min = 0, f_c = 0, df = 0;
  // time samples at the end of each row the detector leaves out at this DM
  size_t reserved(float dm) const {
    return srtb_b200_nsamps_reserved(N, cfg->spectrum_channel_count, cfg->baseband_freq_low, cfg->baseband_bandwidth,
                                     cfg->baseband_sample_rate, dm, cfg->baseband_reserve_sample) /
           batch;
  }
  // s1 + chirp at this DM, applied as a waterfall kernel loads the spectrum
  row_chirp_params chirp(float dm, const float* mean) const {
    constexpr double D = 4.148808e3;  // coherent_dedispersion.hpp:67
    return {(double)f_min, (double)df, 1.0 / (double)f_c, (double)f_c, (D * 1e6) * (double)dm,
            mean, cfg->mitigate_rfi_average_method_threshold, coef, 0};
  }
  // row s (a stream, or the sum after the streams) of a block's pinned series [rows][MAX_BOXCARS][L], or null without
  float* series_row(float* h_series, int s) const {
    return h_series ? h_series + (size_t)s * SRTB_B200_MAX_BOXCARS * L : nullptr;
  }
};

static int block_params_for(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg, const char* who, block_params* p) {
  p->cfg = cfg;
  p->streams = format_streams(cfg->baseband_format);
  if (!p->streams) return fail(ctx, SRTB_B200_E_UNSUPPORTED, std::string(who) + ": unknown format");
  if (cfg->signal_detect_sum_streams && p->streams < 2)
    return fail(ctx, SRTB_B200_E_INVALID,
                std::string(who) + ": signal_detect_sum_streams needs a format with two or more streams");
  p->N = cfg->baseband_input_count;
  if (p->N < 2 || !is_pow2(p->N))
    return fail(ctx, SRTB_B200_E_SIZE, "[fft] n must be a power of 2, got " + std::to_string(p->N));
  p->Nc = p->N / 2;
  p->batch = std::min<size_t>(cfg->spectrum_channel_count, p->Nc);  // fft_pipe.hpp:318-320
  if (p->batch == 0 || !is_pow2(p->batch))
    return fail(ctx, SRTB_B200_E_SIZE, "spectrum_channel_count must be a power of 2");
  p->L = p->Nc / p->batch;
  // manual zap ranges -> bins (host, rfi_mitigation.hpp:102-143)
  for (uint64_t r = 0; r < cfg->n_rfi_freq_pairs; r++) {
    size_t lo, hi;
    if (srtb_b200_rfi_range_to_bins(cfg->rfi_freq_pairs[2 * r], cfg->rfi_freq_pairs[2 * r + 1],
                                    cfg->baseband_freq_low, cfg->baseband_bandwidth, p->Nc, &lo, &hi)) {
      p->bins.push_back(lo);
      p->bins.push_back(hi);
    }
  }
  p->coef = srtb_b200_norm_coefficient(p->Nc, cfg->spectrum_channel_count);
  p->df = cfg->baseband_bandwidth / static_cast<float>(p->Nc);  // dedisperse_pipe.hpp:34
  p->f_min = cfg->baseband_freq_low;
  p->f_c = p->f_min + cfg->baseband_bandwidth;
  return 0;
}

// the block's baseband on the device and the per-stream buffers its R2C writes; raw[] describes the bytes for the
// route with the unpack fused into the first sweep
struct block_input {
  const void* d_baseband;
  size_t bytes;
  float* const* bufs;
  raw_source raw[4];
  bool fuse_unpack = false, unpacked = false;
};

static int unpack_block(srtb_b200_ctx* ctx, const block_params& p, block_input* in) {
  if (in->unpacked) return 0;
  in->unpacked = true;
  return srtb_b200_unpack(ctx, in->d_baseband, in->bytes, p.cfg->baseband_input_bits, p.cfg->baseband_format,
                          p.cfg->window, in->bufs, p.N);
}

// the fused route when the format allows it, else the unpack kernel for every stream now
static int block_input_init(srtb_b200_ctx* ctx, const block_params& p, block_input* in) {
  in->fuse_unpack = raw_sources_for(p.cfg, in->d_baseband, in->bytes, p.streams, in->raw);
  return in->fuse_unpack ? 0 : unpack_block(ctx, p, in);
}

// The sweep-order route of 2^25-point R2Cs with rows of 2^14 (config #3): M = P Q, P = 2^11, Q = L = 2^14. Sweep 1 is the
// raw-fused 2^11-point column sweep into the lane's scratch, sweep 2 the R2C row sweep (2^14-point rows, split, Σ|X|^2)
// from the scratch into the stream's buffer, channel-blocked: bin k = k1 + P k2 sits at (k2 >> 3) Q + 8 k1 + (k2 & 7),
// so channel c (L = 8 P bins) is one contiguous range, laid out [k1][k2 & 7], and the whole-row waterfall kernel
// transforms it in place (24 bytes per sample per stream instead of 32: no third sweep, no fix-up). Taken when the
// unpack is fused (8-bit samples), the geometry is this one, every buffer is 16-byte aligned and TMA tensor maps can
// be encoded; everything else keeps the three-sweep plan.
constexpr unsigned SWEEP_LOGP = 11, SWEEP_LOGQ = 14;
static bool r2c_sweep_order(const block_params& p, const block_input& in) {
  if (!in.fuse_unpack || in.raw[0].bits != 0 || p.L != ((size_t)1 << SWEEP_LOGQ) ||
      p.Nc != ((size_t)1 << (SWEEP_LOGP + SWEEP_LOGQ)) || !get_encode_tiled())
    return false;
  if (reinterpret_cast<uintptr_t>(in.raw[0].base) & 15u) return false;
  for (int s = 0; s < p.streams; s++)
    if (reinterpret_cast<uintptr_t>(in.bufs[s]) & 15u) return false;
  return true;
}

static int r2c_sweep_order_stream(srtb_b200_ctx* ctx, const block_params& p, const block_input& in, int s,
                                  float2* spectrum) {
  const size_t P = (size_t)1 << SWEEP_LOGP, Q = (size_t)1 << SWEEP_LOGQ;
  if (int rc = grow(ctx, ctx->lane.fft_scratch, P * Q * sizeof(float2))) return rc;
  float2* const z = ctx->lane.fft_scratch.p;
  bool done = false;
  if (int rc = dispatch_col_raw(ctx, (int)SWEEP_LOGP, in.raw[s], z, Q, &done)) return rc;
  if (!done) return fail(ctx, SRTB_B200_E_UNSUPPORTED, "r2c: the raw 2^11-point column sweep refused the block");
  return launch_r2c_rows(ctx, z, spectrum, P);
}

// R2C of stream s in its buffer, leaving mean(|X|^2) in the lane's `mean`. When the fused route refuses this size or
// alignment, all streams are unpacked once and take the plain R2C. The route is a property of the block (same size and
// base pointer for every stream), so it can only change on stream 0; later it would overwrite finished streams with
// their unpacked input. fork: the second lane must see the unpacked samples, so it is forked again after that unpack.
static int r2c_stream(srtb_b200_ctx* ctx, const block_params& p, block_input* in, int s, bool fork) {
  float* buf = in->bufs[s];
  if (in->fuse_unpack && !in->unpacked) {
    const int rc = fft_r2c_with_power_mean(ctx, buf, p.N, &in->raw[s], nullptr);
    if (rc != SRTB_B200_E_UNSUPPORTED) return rc;
    if (s > 0)
      return fail(ctx, SRTB_B200_E_UNSUPPORTED,
                  "fused unpack refused stream " + std::to_string(s) + " after accepting stream 0");
    if (int rc2 = unpack_block(ctx, p, in)) return rc2;
    if (fork)
      if (int rc2 = fork_lanes(ctx)) return rc2;
  }
  return fft_r2c_with_power_mean(ctx, buf, p.N);
}

// routes that apply s1 + the chirp as a waterfall kernel loads the spectrum: the caller zaps the manual ranges on the
// spectrum beforehand (0 stays 0 through s1 and the chirp)
static bool chirp_on_load(size_t L) { return chirp_fusable(L) || long_fusable(L); }

// one stream's chain after its R2C, at one DM: s1 + chirp, waterfall FFT, SK and detector writing to `out`. src holds the spectrum, dst receives the dynamic spectrum: the same buffer on the block path, while the
// DM sweep keeps src for the next trial. phase_table: the whole-row kernel may read a tabulated chirp (built for the
// block's DM; the DM sweep changes DM every trial). sweep_order: src is the channel-blocked spectrum of r2c_sweep_order,
// whose waterfall kernel evaluates every phase itself. Both buffers are 16-byte aligned: the ctx allocates them, or
// submit_block_ex checked the caller's.
static int stream_tail(srtb_b200_ctx* ctx, const block_params& p, const detect_out& out, float2* dst, const float2* src, float dm,
                       bool phase_table, bool sweep_order = false) {
  const srtb_b200_block_config* cfg = p.cfg;
  const size_t reserved = p.reserved(dm);
  if (chirp_fusable(p.L)) {
    // ONE kernel: s1 + chirp on load, waterfall FFT, SK, partial column sums
    row_chirp_params cp = p.chirp(dm, ctx->lane.mean);
    if (phase_table)
      if (int rc = get_chirp_table(ctx, p.Nc, cp, &cp.phase)) return rc;
    return watfft_sk_detect_fused(ctx, out, dst, p.L, p.batch, reserved, cfg->mitigate_rfi_spectral_kurtosis_threshold,
                                  cfg->signal_detect_signal_noise_threshold, cfg->signal_detect_channel_threshold,
                                  cfg->signal_detect_max_boxcar_length, &cp, src, sweep_order);
  }
  if (long_fusable(p.L)) {
    // long rows: chirp-on-load column sweep, last sweep with SK statistics, decision, column sums (20 bytes per
    // sample). No phase table here: the long-row column sweep is DRAM-bound, and the 4 extra bytes per bin a table
    // costs outweigh the fp64 evaluation it would replace.
    const int rc = watfft_long_fused(ctx, out, dst, src, p.L, p.batch, reserved,
                                     cfg->mitigate_rfi_spectral_kurtosis_threshold,
                                     cfg->signal_detect_signal_noise_threshold, cfg->signal_detect_channel_threshold,
                                     cfg->signal_detect_max_boxcar_length, p.chirp(dm, ctx->lane.mean));
    if (rc != SRTB_B200_E_UNSUPPORTED) return rc;
  }
  if (int rc = rfi_s1_dedisperse_fused(ctx, dst, src, p.Nc, cfg->mitigate_rfi_average_method_threshold, p.coef, p.bins,
                                       p.f_min, p.f_c, p.df, dm))
    return rc;
  if (p.L == 512) {
    // waterfall FFT + SK + partial column sums in one kernel (the eight-point row kernel has no chirp on load), then
    // the small detector tail
    return watfft_sk_detect_fused(ctx, out, dst, p.L, p.batch, reserved, cfg->mitigate_rfi_spectral_kurtosis_threshold,
                                  cfg->signal_detect_signal_noise_threshold, cfg->signal_detect_channel_threshold,
                                  cfg->signal_detect_max_boxcar_length);
  }
  if (int rc = srtb_b200_watfft_c2c_backward(ctx, dst, p.L, p.batch)) return rc;
  if (int rc = srtb_b200_rfi_s2_sk(ctx, dst, p.L, p.batch, cfg->mitigate_rfi_spectral_kurtosis_threshold, nullptr))
    return rc;
  return detect_enqueue(ctx, out, dst, p.L, p.batch, reserved, cfg->signal_detect_signal_noise_threshold,
                        cfg->signal_detect_channel_threshold, cfg->signal_detect_max_boxcar_length);
}

// the detector on the total intensity of the block's streams (stream_sum.cuh), on the first lane once every stream's
// chain has run: mask, sum, then the detector's tail on the summed series, header in d_res[SUM_SLOT]. raw: the streams'
// raw column sums [4][L]; host_series (optional): the block's pinned series, whose slot `streams` receives the sum's
// positive series
static int sum_tail(srtb_b200_ctx* ctx, const block_params& p, float* const* bufs, const float* raw,
                    float* host_series) {
  const srtb_b200_block_config* cfg = p.cfg;
  const size_t L = p.L, C = p.batch;
  const size_t ts = detected_samples(L, p.reserved(cfg->dm));
  if (int rc = detect_prepare(ctx, SUM_SLOT, L, 1)) return rc;
  if (int rc = grow(ctx, ctx->sum_mask, C * (sizeof(float2) + sizeof(uint2)) + sizeof(unsigned))) return rc;
  float2* const mask = ctx->sum_mask.p;
  uint2* const mis = reinterpret_cast<uint2*>(mask + C);
  unsigned* const n_mis = reinterpret_cast<unsigned*>(mis + C);
  stream_sum_inputs in{};
  for (int s = 0; s < p.streams; s++) {
    in.x[s] = reinterpret_cast<const float2*>(bufs[s]);
    in.raw[s] = raw + (size_t)s * L;
  }
  CK(cudaMemsetAsync(ctx->d_res + SUM_SLOT, 0, sizeof(detect_dev_result), ctx->lane.stream));
  CK(launch(ctx, false, stream_sum_mask_kernel, 1, 1024, 0, in, p.streams, L, C, mask, mis, n_mis));
  CK(launch(ctx, true, stream_sum_kernel, grid_for(ctx, ts, 256), 256, 0, in, p.streams, L, ts, (const uint2*)mis,
            (const unsigned*)n_mis, ctx->series[SUM_SLOT].p));
  // the tail counts the mask's zeros (stride 1): the union count. The first lane's ticket and scan buffer are free here:
  // its own stream's tail has finished in stream order.
  const detect_out out{SUM_SLOT, p.series_row(host_series, p.streams), nullptr, nullptr, /*header_zeroed=*/true};
  return detect_tail(ctx, out, nullptr, mask, L, C, ts, 0, cfg->signal_detect_signal_noise_threshold,
                     cfg->signal_detect_channel_threshold, cfg->signal_detect_max_boxcar_length, /*zero_stride=*/1);
}

// ---- events: every above-threshold run of a detector's series (events.cuh), found by two launches that write into a
// pinned ev_list through a lane's scratch. The block path (srtb_b200_submit_block_events) runs them at the end of every
// detector's own chain, on its lane, into the ring slot's list; the DM searches and series_events run them on the
// first lane into ctx->ev_host. A lane's scratch serves one pass at a time in stream order.
struct ev_scratch {
  unsigned long long* count;   // [RES_GROUP] running counts, at the head
  unsigned* ticket;            // the count kernel's, at the head
  ev_tile* tile;               // [n_rec][max_nb][tiles] tile summaries
  unsigned long long* offset;  // their scan offsets
  detect_dev_result* headers;  // uploaded headers
  unsigned max_nb;             // boxcar rows per record the launches cover
  size_t tiles;                // tiles of EV_TILE samples per row
};

// lane l's scratch for n_rec records of max_nb rows of at most row_len samples, and n_headers uploaded headers: the
// head (EV_HEAD bytes), the tile summaries, their offsets and the headers, each 256-byte aligned
static int ev_scratch_for(srtb_b200_ctx* ctx, lane_state& l, const char* who, size_t n_rec, unsigned max_nb,
                          size_t row_len, size_t n_headers, ev_scratch* sc) {
  const size_t tiles = std::max<size_t>(1, (row_len + EV_TILE - 1) / EV_TILE);
  const size_t nt = n_rec * max_nb * tiles;
  if (n_rec > 65535 || tiles > 0x7fffffffu || nt >= ((size_t)1 << 32))
    return fail(ctx, SRTB_B200_E_SIZE, std::string(who) + ": too many tiles for the event pass");
  const size_t off_o = EV_HEAD + ((nt * sizeof(ev_tile) + 255) & ~(size_t)255);
  const size_t hdr_o = off_o + ((nt * sizeof(unsigned long long) + 255) & ~(size_t)255);
  if (int rc = grow(ctx, l.ev_work, hdr_o + n_headers * sizeof(detect_dev_result))) return rc;
  char* const w = l.ev_work.p;
  *sc = ev_scratch{reinterpret_cast<unsigned long long*>(w),
                   reinterpret_cast<unsigned*>(w + RES_GROUP * sizeof(unsigned long long)),
                   reinterpret_cast<ev_tile*>(w + EV_HEAD), reinterpret_cast<unsigned long long*>(w + off_o),
                   reinterpret_cast<detect_dev_result*>(w + hdr_o), max_nb, tiles};
  return 0;
}

// zeroes the scratch's counts and ticket on the current lane: at the head of a chain, never between two of its kernels
static int ev_zero(srtb_b200_ctx* ctx, const ev_scratch& sc) {
  CK(cudaMemsetAsync(sc.count, 0, EV_HEAD, ctx->lane.stream));
  return 0;
}

// b holds a list of `rows` rows of max_events afterwards
static int ev_list_for(srtb_b200_ctx* ctx, buffer<char, true>& b, size_t rows, size_t max_events, ev_list* list) {
  if (int rc = grow(ctx, b, EV_HEAD + rows * std::max<size_t>(max_events, 1) * sizeof(ev_event))) return rc;
  *list = ev_list{b.p, max_events};
  return 0;
}

// the two event launches over n_rec records (rows as r describes them), counting from *count (the ticket zero), into
// list row r.stream
static int events_enqueue(srtb_b200_ctx* ctx, const ev_scratch& sc, const ev_rows& r, size_t n_rec,
                          unsigned long long* count, const ev_list& list) {
  const dim3 grid((unsigned)r.tiles, r.max_nb, (unsigned)n_rec);
  CK(launch(ctx, false, ev_count_kernel, grid, EV_THREADS, 0, r, sc.tile, sc.offset, sc.ticket, count));
  CK(launch(ctx, false, ev_emit_kernel, grid, EV_THREADS, 0, r, (const ev_tile*)sc.tile,
            (const unsigned long long*)sc.offset, list.row(r.stream), (unsigned long long)list.max_events));
  return 0;
}

// after detector `slot` (a stream, or SUM_SLOT) has run on the current lane, whose scratch is sc: its events, as list
// row `row` with stream = row, and their count into the list's head
static int block_ev_enqueue(srtb_b200_ctx* ctx, const ev_scratch& sc, const ev_list& list, int slot, size_t L,
                            unsigned row) {
  const ev_rows r{ctx->series[slot].p, L, 0, ctx->d_res + slot, sc.max_nb, sc.tiles, 0u, row};
  if (int rc = events_enqueue(ctx, sc, r, 1, sc.count + slot, list)) return rc;
  CK(cudaMemcpyAsync(list.counts() + row, sc.count + slot, sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                     ctx->lane.stream));
  return 0;
}

// enqueue every stage of one block (no host sync); results land in ctx->h_res[res_base .. res_base + streams) once the
// lanes reach their D2H copies. bufs[s]: working buffer of stream s (N + 2 floats, 16-byte aligned for the fused
// routes), which holds the dynamic spectrum [C][L] when the block is done. host_series (optional): pinned host memory
// that receives positive series. join_lanes: the first lane waits for the second at the end (process_block); the ring
// leaves the lanes free-running (each copies its own result headers back, *alt_used tells the caller to record a
// completion event on both). With cfg->signal_detect_sum_streams the first lane then waits for the second on the device
// and runs sum_tail; its header lands in h_res[res_base + SUM_SLOT]. ev (the ring slot's list for the events entry, or
// null): every detector's events after its tail, on its lane (two launches and a count copy per stream, and per sum).
static int block_enqueue(srtb_b200_ctx* ctx, const block_params& p, const void* d_baseband, size_t baseband_bytes,
                         int res_base, float* const* bufs, float* host_series, bool join_lanes = true,
                         bool* alt_used = nullptr, const ev_list* ev = nullptr) {
  struct pdl_scope {  // launch reads ctx->pdl_auto; it is only meaningful inside this call
    srtb_b200_ctx* c;
    ~pdl_scope() { c->pdl_auto = false; }
  } pdl_scope_{ctx};
  ctx->pdl_auto = p.N <= ((size_t)1 << 25);
  const bool sum = p.cfg->signal_detect_sum_streams != 0;
  float* raw = nullptr;  // this block's raw column sums [4][L]
  if (sum) {
    const size_t group = (size_t)(res_base / RES_GROUP);
    if (int rc = grow(ctx, ctx->sum_raw, (1 + SRTB_B200_RING_SLOTS) * 4 * p.L * sizeof(float))) return rc;
    raw = ctx->sum_raw.p + group * 4 * p.L;
  }
  // the data streams of a block are independent: odd ones go to the context's second lane (per-stage timing wants the
  // kernels alone, so it keeps one lane)
  const bool two_lanes = ctx->lanes >= 2 && p.streams >= 2 && !ctx->stats_on;
  if (alt_used) *alt_used = two_lanes;
  if (two_lanes) {
    if (int rc = ensure_alt_lane(ctx)) return rc;
  }
  ev_scratch evs[2] = {};  // the first lane's event scratch, the second's: one detector's rows of L
  if (ev) {
    const unsigned max_nb = boxcar_ctas(p.cfg->signal_detect_max_boxcar_length, p.L);
    if (int rc = ev_scratch_for(ctx, ctx->lane, "submit_block_events", 1, max_nb, p.L, 0, &evs[0])) return rc;
    if (two_lanes)
      if (int rc = ev_scratch_for(ctx, ctx->alt, "submit_block_events", 1, max_nb, p.L, 0, &evs[1])) return rc;
  }
  if (!two_lanes) {
    // result headers zeroed before the first kernel (a memset between kernels would break the dependent-launch chain);
    // with two lanes every stream zeroes its own header at the head of its chain, on its lane. The event counts alike.
    CK(cudaMemsetAsync(ctx->d_res, 0, sizeof(detect_dev_result) * p.streams, ctx->lane.stream));
    if (ev)
      if (int rc = ev_zero(ctx, evs[0])) return rc;
  }
  block_input in{d_baseband, baseband_bytes, bufs};
  if (int rc = block_input_init(ctx, p, &in)) return rc;
  if (two_lanes)
    if (int rc = fork_lanes(ctx)) return rc;
  const bool sweep_order = r2c_sweep_order(p, in);
  auto enqueue_stream = [&](int s) -> int {
    float2* buf = reinterpret_cast<float2*>(bufs[s]);
    if (two_lanes) {
      CK(cudaMemsetAsync(ctx->d_res + s, 0, sizeof(detect_dev_result), ctx->lane.stream));
      if (ev)
        if (int rc = ev_zero(ctx, evs[s & 1])) return rc;
    }
    const detect_out out{s, p.series_row(host_series, s), raw ? raw + (size_t)s * p.L : nullptr, nullptr,
                         /*header_zeroed=*/true};
    if (sweep_order) {
      {
        stage_scope stats_(ctx, SRTB_B200_STAGE_FUSED_R2C,
                           (double)p.N * (double)std::abs(p.cfg->baseband_input_bits) / 8.0 + 4.0 * (double)p.N);
        if (int rc = r2c_sweep_order_stream(ctx, p, in, s, buf)) return rc;
      }
      if (int rc = zero_bin_ranges(ctx, buf, p.bins, SWEEP_LOGP, SWEEP_LOGQ)) return rc;
      return stream_tail(ctx, p, out, buf, buf, p.cfg->dm, /*phase_table=*/false, /*sweep_order=*/true);
    }
    {
      stage_scope stats_(ctx, SRTB_B200_STAGE_FUSED_R2C,
                         (double)p.N * (in.fuse_unpack ? (double)std::abs(p.cfg->baseband_input_bits) / 8.0 : 4.0) +
                             4.0 * (double)p.N);
      if (int rc = r2c_stream(ctx, p, &in, s, /*fork=*/two_lanes)) return rc;
    }
    if (chirp_on_load(p.L))
      if (int rc = zero_bin_ranges(ctx, buf, p.bins)) return rc;
    return stream_tail(ctx, p, out, buf, buf, p.cfg->dm, /*phase_table=*/true);
  };
  for (int s = 0; s < p.streams; s++) {
    const bool alt = two_lanes && (s & 1);
    if (alt) lane_swap(ctx);
    int rc = enqueue_stream(s);
    // every route of stream_tail ends in detect_tail, which leaves series[s] and d_res[s] for the event pass
    if (!rc && ev) rc = block_ev_enqueue(ctx, evs[alt], *ev, s, p.L, (unsigned)s);
    if (!rc && two_lanes) {
      const cudaError_t e = cudaMemcpyAsync(ctx->h_res + res_base + s, ctx->d_res + s, sizeof(detect_dev_result),
                                            cudaMemcpyDeviceToHost, ctx->lane.stream);
      if (e != cudaSuccess) rc = fail(ctx, SRTB_B200_E_CUDA, std::string("result header copy: ") + cudaGetErrorString(e));
    }
    if (alt) lane_swap(ctx);
    if (rc) return rc;
  }
  if (two_lanes && (join_lanes || sum)) {
    CK(cudaEventRecord(ctx->lane_join, ctx->alt.stream));
    CK(cudaStreamWaitEvent(ctx->lane.stream, ctx->lane_join, 0));
  }
  if (!two_lanes)
    CK(cudaMemcpyAsync(ctx->h_res + res_base, ctx->d_res, sizeof(detect_dev_result) * p.streams, cudaMemcpyDeviceToHost,
                       ctx->lane.stream));
  if (sum) {
    if (ev)  // the sum's chain head, next to sum_tail's header memset
      if (int rc = ev_zero(ctx, evs[0])) return rc;
    if (int rc = sum_tail(ctx, p, bufs, raw, host_series)) return rc;
    if (ev)
      if (int rc = block_ev_enqueue(ctx, evs[0], *ev, SUM_SLOT, p.L, (unsigned)p.streams)) return rc;
    CK(cudaMemcpyAsync(ctx->h_res + res_base + SUM_SLOT, ctx->d_res + SUM_SLOT, sizeof(detect_dev_result),
                       cudaMemcpyDeviceToHost, ctx->lane.stream));
  }
  return 0;
}

// the caller's spectra (d_spectrum of the block or sweep outputs, or null): given for every stream or for none, each
// 16-byte aligned. *given: they are.
static int caller_spectra(srtb_b200_ctx* ctx, const char* who, float* const* d_spectrum, int streams, bool* given) {
  *given = d_spectrum && d_spectrum[0];
  for (int s = 0; d_spectrum && s < streams; s++) {
    if (!d_spectrum[s] == *given)
      return fail(ctx, SRTB_B200_E_INVALID, std::string(who) + ": d_spectrum given for some streams only");
    if (*given && !aligned16(d_spectrum[s]))
      return fail(ctx, SRTB_B200_E_INVALID,
                  std::string(who) + ": d_spectrum[" + std::to_string(s) + "] is not 16-byte aligned");
  }
  return 0;
}

// the block's baseband on the device: the caller's (on_device), else the host bytes copied into ctx->d_baseband on the
// current lane
static int device_baseband(srtb_b200_ctx* ctx, const void* baseband, size_t bytes, int on_device, const void** d) {
  *d = baseband;
  if (on_device) return 0;
  if (int rc = grow(ctx, ctx->d_baseband, bytes)) return rc;
  CK(cudaMemcpyAsync(ctx->d_baseband.p, baseband, bytes, cudaMemcpyHostToDevice, ctx->lane.stream));
  *d = ctx->d_baseband.p;
  return 0;
}

// bufs[s]: stream s's working buffer of N + 2 floats from own[s] (the ctx's, or a ring slot's), grown for the block
static int own_stream_bufs(srtb_b200_ctx* ctx, const block_params& p, buffer<float>* own, float** bufs) {
  for (int s = 0; s < p.streams; s++) {
    if (int rc = grow(ctx, own[s], (p.N + 2) * sizeof(float))) return rc;
    bufs[s] = own[s].p;
  }
  return 0;
}

extern "C" int srtb_b200_process_block_device(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg,
                                              const void* d_baseband, size_t baseband_bytes,
                                              srtb_b200_detect_result* h_results, float* h_series,
                                              int copy_all) {
  API_LOCK(ctx);
  if (!ctx || !cfg || !d_baseband || !h_results) return fail(ctx, SRTB_B200_E_INVALID, "process_block: null argument");
  CK(cudaSetDevice(ctx->device));
  block_params p;
  if (int rc = block_params_for(ctx, cfg, "process_block", &p)) return rc;
  float* bufs[4] = {};
  if (int rc = own_stream_bufs(ctx, p, ctx->stream_buf, bufs)) return rc;
  if (int rc = block_enqueue(ctx, p, d_baseband, baseband_bytes, 0, bufs, nullptr)) return rc;
  CK(cudaStreamSynchronize(ctx->lane.stream));
  for (int s = 0; s < p.streams; s++)
    if (int rc = detect_collect(ctx, s, h_results + s, p.series_row(h_series, s), copy_all)) return rc;
  if (cfg->signal_detect_sum_streams)
    if (int rc = detect_collect(ctx, SUM_SLOT, h_results + p.streams, p.series_row(h_series, p.streams), copy_all))
      return rc;
  return p.streams;
}

extern "C" int srtb_b200_process_block(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg,
                                       const void* h_baseband, size_t baseband_bytes,
                                       srtb_b200_detect_result* h_results, float* h_series, int copy_all) {
  API_LOCK(ctx);
  if (!ctx || !cfg || !h_baseband) return fail(ctx, SRTB_B200_E_INVALID, "process_block: null argument");
  CK(cudaSetDevice(ctx->device));
  const void* d_baseband = nullptr;
  if (int rc = device_baseband(ctx, h_baseband, baseband_bytes, /*on_device=*/0, &d_baseband)) return rc;
  return srtb_b200_process_block_device(ctx, cfg, d_baseband, baseband_bytes, h_results, h_series, copy_all);
}

// ---- events: every above-threshold run of the detector's series (events.cuh) -----------------------------------------

// where a DM search's events go: max_events per stream into h_events, the totals into n_events[streams]
struct ev_request {
  srtb_b200_event* h_events;
  size_t max_events;
  uint64_t* n_events;
};

// the event pass of one synchronous call, before any of its launches: the first lane's scratch (ev_scratch_for), with its
// counts zeroed, and ctx->ev_host as the list of `streams` rows of max_events
static int events_prepare(srtb_b200_ctx* ctx, const char* who, size_t n_rec, unsigned max_nb, size_t row_len,
                          int streams, size_t max_events, size_t n_headers, ev_scratch* sc, ev_list* list) {
  if (int rc = ev_scratch_for(ctx, ctx->lane, who, n_rec, max_nb, row_len, n_headers, sc)) return rc;
  if (int rc = ev_list_for(ctx, ctx->ev_host, (size_t)streams, max_events, list)) return rc;
  return ev_zero(ctx, *sc);
}

// enqueued before the call's synchronisation: the streams' counts into the list's head
static int events_fetch_counts(srtb_b200_ctx* ctx, const ev_scratch& sc, const ev_list& list, int streams) {
  CK(cudaMemcpyAsync(list.counts(), sc.count, streams * sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                     ctx->lane.stream));
  return 0;
}

// after the synchronisation: the counts and the written events to the caller
static void events_collect(const ev_list& list, int streams, const ev_request& ev) {
  for (int s = 0; s < streams; s++) {
    ev.n_events[s] = list.counts()[s];
    const size_t k = (size_t)std::min<unsigned long long>(list.counts()[s], ev.max_events);
    if (k) std::memcpy(ev.h_events + (size_t)s * ev.max_events, list.row(s), k * sizeof(ev_event));
  }
}

static bool ev_request_ok(const ev_request* ev) {
  return !ev || (ev->n_events && (ev->h_events || ev->max_events == 0));
}

extern "C" int srtb_b200_series_events(srtb_b200_ctx* ctx, const float* d_series, size_t boxcar_stride,
                                       size_t trial_stride, const srtb_b200_detect_result* h_results, size_t n_trials,
                                       srtb_b200_event* h_events, size_t max_events, uint64_t* n_events) {
  API_LOCK(ctx);
  const ev_request ev{h_events, max_events, n_events};
  if (!ctx || !d_series || !h_results || !ev_request_ok(&ev) || n_trials == 0 || n_trials > 65535)
    return fail(ctx, SRTB_B200_E_INVALID, "series_events: bad argument");
  unsigned max_nb = 0;
  size_t row_len = 0;
  for (size_t y = 0; y < n_trials; y++) {
    const srtb_b200_detect_result& r = h_results[y];
    if (r.n_boxcars < 0 || r.n_boxcars > SRTB_B200_MAX_BOXCARS)
      return fail(ctx, SRTB_B200_E_INVALID, "series_events: n_boxcars outside 0..32");
    if (!r.detect_enabled) continue;
    max_nb = std::max(max_nb, (unsigned)r.n_boxcars);
    size_t extent = 0;  // of the trial's rows
    for (int b = 0; b < r.n_boxcars; b++) {
      row_len = std::max<size_t>(row_len, r.series_length[b]);
      extent = std::max<size_t>(extent, (size_t)b * boxcar_stride + r.series_length[b]);
      if (r.n_boxcars > 1 && r.series_length[b] > boxcar_stride)
        return fail(ctx, SRTB_B200_E_INVALID, "series_events: a row is longer than boxcar_stride");
    }
    if (n_trials > 1 && extent > trial_stride)
      return fail(ctx, SRTB_B200_E_INVALID, "series_events: a trial's rows are longer than trial_stride");
  }
  CK(cudaSetDevice(ctx->device));
  ev_scratch sc;
  ev_list list;
  if (int rc = events_prepare(ctx, "series_events", n_trials, std::max(max_nb, 1u), row_len, 1, max_events, n_trials,
                              &sc, &list))
    return rc;
  CK(cudaMemcpyAsync(sc.headers, h_results, n_trials * sizeof(detect_dev_result), cudaMemcpyHostToDevice,
                     ctx->lane.stream));
  if (max_nb > 0) {
    const ev_rows r{d_series, boxcar_stride, trial_stride, sc.headers, max_nb, sc.tiles, 0u, 0u};
    if (int rc = events_enqueue(ctx, sc, r, n_trials, sc.count, list)) return rc;
  }
  if (int rc = events_fetch_counts(ctx, sc, list, 1)) return rc;
  CK(cudaStreamSynchronize(ctx->lane.stream));
  events_collect(list, 1, ev);
  return 0;
}

// friends of friends over the events (include/srtb_b200.h): union-find, joined by one sweep over the spans per stream
extern "C" int srtb_b200_cluster_events(const srtb_b200_event* h_events, size_t n_events, const float* h_dms,
                                        size_t n_dm, srtb_b200_candidate* h_candidates, size_t max_candidates,
                                        uint64_t* n_candidates) {
  if (!n_candidates || (!h_events && n_events) || !h_dms || n_dm == 0 || (!h_candidates && max_candidates))
    return fail(nullptr, SRTB_B200_E_INVALID, "cluster_events: bad argument");
  for (size_t i = 0; i < n_events; i++) {
    const srtb_b200_event& e = h_events[i];
    if (e.trial >= n_dm || e.boxcar > 31 || e.end <= e.begin)
      return fail(nullptr, SRTB_B200_E_INVALID, "cluster_events: event " + std::to_string(i) + " is malformed");
  }
  std::vector<uint32_t> rank(n_dm), order(n_dm);
  for (size_t d = 0; d < n_dm; d++) order[d] = (uint32_t)d;
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return h_dms[a] < h_dms[b]; });
  for (size_t r = 0; r < n_dm; r++) rank[order[r]] = (uint32_t)r;
  auto o_of = [](const srtb_b200_event& e) -> uint64_t { return e.boxcar ? 1 : 0; };
  auto lo_of = [&](const srtb_b200_event& e) { return e.begin + o_of(e); };
  auto hi_of = [&](const srtb_b200_event& e) { return e.end - 1 + o_of(e) + ((uint64_t)1 << e.boxcar); };
  std::vector<size_t> parent(n_events);
  for (size_t i = 0; i < n_events; i++) parent[i] = i;
  auto find = [&](size_t i) {
    while (parent[i] != i) {
      parent[i] = parent[parent[i]];
      i = parent[i];
    }
    return i;
  };
  auto unite = [&](size_t a, size_t b) {
    a = find(a);
    b = find(b);
    if (a != b) parent[std::max(a, b)] = std::min(a, b);
  };
  // sweep by (stream, span begin): every active event of a rank contains the sweep point, so those of one rank are
  // friends of each other and of the event at the sweep point when the ranks are at most 1 apart. One active event per
  // rank (the one whose span ends last) stands for all of them.
  std::vector<size_t> by(n_events);
  for (size_t i = 0; i < n_events; i++) by[i] = i;
  std::sort(by.begin(), by.end(), [&](size_t a, size_t b) {
    const srtb_b200_event &x = h_events[a], &y = h_events[b];
    if (x.stream != y.stream) return x.stream < y.stream;
    if (lo_of(x) != lo_of(y)) return lo_of(x) < lo_of(y);
    return a < b;
  });
  std::vector<uint64_t> act_end(n_dm, 0);
  std::vector<size_t> act_id(n_dm, 0);
  std::vector<uint32_t> act_stream(n_dm, ~0u);
  for (size_t i : by) {
    const srtb_b200_event& e = h_events[i];
    const uint64_t x = lo_of(e), end = hi_of(e);
    const uint32_t r = rank[e.trial];
    for (uint32_t q = r ? r - 1 : 0; q <= r + 1 && q < n_dm; q++)
      if (act_stream[q] == e.stream && act_end[q] > x) unite(i, act_id[q]);
    if (act_stream[r] != e.stream || act_end[r] <= x || end > act_end[r]) {
      act_stream[r] = e.stream;
      act_end[r] = end;
      act_id[r] = i;
    }
  }
  // components: representative, members, DM range, span
  std::vector<size_t> comp(n_events, SIZE_MAX);
  std::vector<srtb_b200_candidate> cands;
  std::vector<size_t> rep;  // event index of each candidate's representative
  auto better = [&](const srtb_b200_event& a, const srtb_b200_event& b) {  // a beats b
    if (a.snr != b.snr) return a.snr > b.snr;
    if (a.trial != b.trial) return a.trial < b.trial;
    if (a.boxcar != b.boxcar) return a.boxcar < b.boxcar;
    return a.begin < b.begin;
  };
  for (size_t i = 0; i < n_events; i++) {
    const size_t root = find(i);
    const srtb_b200_event& e = h_events[i];
    const float dm = h_dms[e.trial];
    if (comp[root] == SIZE_MAX) {
      comp[root] = cands.size();
      srtb_b200_candidate c{};
      c.dm_low = c.dm_high = dm;
      c.span_begin = lo_of(e);
      c.span_end = hi_of(e);
      c.stream = e.stream;
      cands.push_back(c);
      rep.push_back(i);
    }
    srtb_b200_candidate& c = cands[comp[root]];
    c.members++;
    c.dm_low = std::min(c.dm_low, dm);
    c.dm_high = std::max(c.dm_high, dm);
    c.span_begin = std::min(c.span_begin, lo_of(e));
    c.span_end = std::max(c.span_end, hi_of(e));
    if (better(e, h_events[rep[comp[root]]])) rep[comp[root]] = i;
  }
  for (size_t k = 0; k < cands.size(); k++) {
    const srtb_b200_event& e = h_events[rep[k]];
    srtb_b200_candidate& c = cands[k];
    c.snr = e.snr;
    c.dm = h_dms[e.trial];
    c.trial = e.trial;
    c.boxcar_length = (uint64_t)1 << e.boxcar;
    c.peak_index = e.peak_index;
    c.window = e.peak_index + o_of(e);
  }
  std::vector<size_t> out(cands.size());
  for (size_t k = 0; k < out.size(); k++) out[k] = k;
  std::sort(out.begin(), out.end(), [&](size_t a, size_t b) {
    const srtb_b200_candidate &x = cands[a], &y = cands[b];
    if (x.stream != y.stream) return x.stream < y.stream;
    if (x.span_begin != y.span_begin) return x.span_begin < y.span_begin;
    if (x.trial != y.trial) return x.trial < y.trial;
    if (x.boxcar_length != y.boxcar_length) return x.boxcar_length < y.boxcar_length;
    return h_events[rep[a]].begin < h_events[rep[b]].begin;
  });
  *n_candidates = cands.size();
  for (size_t k = 0; k < std::min(max_candidates, out.size()); k++) h_candidates[k] = cands[out[k]];
  return 0;
}

// ---- DM sweep on one block (BASELINE config #4): unpack + R2C + mean once per stream, then for every
// trial DM the s1-apply + chirp (out of place, the spectrum is kept), waterfall FFT, SK and detector.
// Each trial's result equals process_block with cfg->dm = that DM on the same block.
// With outputs, every trial's detector also writes its peaks, the host picks each stream's best trial, and one more
// stream_tail per stream at that trial's DM writes its dynamic spectrum and positive series.

// the best trial of stream s: among the trials with detection enabled, those with a positive boxcar first, then the
// largest peak S/N over the boxcars, then the lowest index; trial 0 when no trial has detection enabled
static int best_trial(const srtb_b200_detect_result* res, const detect_dev_peak* peaks, size_t n_dm, int streams,
                      int s) {
  int best = -1;
  bool best_positive = false;
  float best_snr = 0.f;
  for (size_t j = 0; j < n_dm; j++) {
    const srtb_b200_detect_result& r = res[j * streams + s];
    if (!r.detect_enabled) continue;
    bool positive = false;
    float snr = -INFINITY;
    for (int b = 0; b < r.n_boxcars; b++) {
      positive = positive || r.signal_count[b] > 0;
      snr = std::max(snr, peaks[j * streams + s].snr[b]);
    }
    if (best < 0 || (positive && !best_positive) || (positive == best_positive && snr > best_snr)) {
      best = (int)j;
      best_positive = positive;
      best_snr = snr;
    }
  }
  return best < 0 ? 0 : best;
}

extern "C" int srtb_b200_process_block_dm_sweep(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg,
                                                const void* baseband, size_t baseband_bytes, int on_device,
                                                const float* h_dms, size_t n_dm,
                                                srtb_b200_detect_result* h_results /* [n_dm][streams] */) {
  return srtb_b200_process_block_dm_sweep_ex(ctx, cfg, baseband, baseband_bytes, on_device, h_dms, n_dm, h_results,
                                             nullptr);
}

// ev (or null): every trial's events, listed by the two event launches after its detector
static int dm_sweep(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg, const void* baseband, size_t baseband_bytes,
                    int on_device, const float* h_dms, size_t n_dm, srtb_b200_detect_result* h_results,
                    const srtb_b200_sweep_outputs* outputs, const ev_request* ev) {
  API_LOCK(ctx);
  if (!ctx || !cfg || !baseband || !h_dms || !h_results || n_dm == 0 || !ev_request_ok(ev))
    return fail(ctx, SRTB_B200_E_INVALID, "dm_sweep: bad argument");
  if (cfg->signal_detect_sum_streams)
    return fail(ctx, SRTB_B200_E_UNSUPPORTED, "dm_sweep: signal_detect_sum_streams is not supported by the DM sweep");
  CK(cudaSetDevice(ctx->device));
  block_params p;
  if (int rc = block_params_for(ctx, cfg, "dm_sweep", &p)) return rc;
  bool user_spec = false;
  if (int rc = caller_spectra(ctx, "dm_sweep", outputs ? outputs->d_spectrum : nullptr, p.streams, &user_spec))
    return rc;
  const void* d_baseband = nullptr;
  if (int rc = device_baseband(ctx, baseband, baseband_bytes, on_device, &d_baseband)) return rc;
  float* bufs[4] = {};
  if (int rc = own_stream_bufs(ctx, p, ctx->stream_buf, bufs)) return rc;
  if (int rc = grow(ctx, ctx->sweep_buf, (p.Nc + 1) * sizeof(float2))) return rc;
  float2* W = ctx->sweep_buf.p;
  // every trial's result header is parked on the device and fetched once at the end: no host sync per trial. With
  // outputs, the trials' peak records [n_dm][streams] follow the headers in the same allocation, then each stream's
  // mean(|X|^2), which s1 reads from the lane and the next stream's R2C overwrites
  const size_t n_rec = n_dm * p.streams;
  if (int rc = grow(ctx, ctx->sweep_res,
                    n_rec * (sizeof(detect_dev_result) + (outputs ? sizeof(detect_dev_peak) : 0)) +
                        (outputs ? 4 * sizeof(float) : 0)))
    return rc;
  detect_dev_result* d_sweep = ctx->sweep_res.p;
  detect_dev_peak* const d_peaks = outputs ? reinterpret_cast<detect_dev_peak*>(d_sweep + n_rec) : nullptr;
  float* const d_means = outputs ? reinterpret_cast<float*>(d_peaks + n_rec) : nullptr;
  // zeroed once before the first kernel: a memset between kernels would break the dependent-launch chain
  if (outputs) CK(cudaMemsetAsync(d_peaks, 0, n_rec * sizeof(detect_dev_peak), ctx->lane.stream));
  // events: rows of at most L samples and boxcar_ctas(max, L) boxcars per trial, one trial per launch pair
  ev_scratch sc{};
  ev_list list;
  const unsigned ev_nb = boxcar_ctas(cfg->signal_detect_max_boxcar_length, p.L);
  if (ev)
    if (int rc = events_prepare(ctx, "dm_sweep", 1, ev_nb, p.L, p.streams, ev->max_events, 0, &sc, &list)) return rc;
  block_input in{d_baseband, baseband_bytes, bufs};
  if (int rc = block_input_init(ctx, p, &in)) return rc;
  for (int s = 0; s < p.streams; s++) {
    if (int rc = r2c_stream(ctx, p, &in, s, /*fork=*/false)) return rc;
    if (d_means)
      CK(cudaMemcpyAsync(d_means + s, ctx->lane.mean, sizeof(float), cudaMemcpyDeviceToDevice, ctx->lane.stream));
    float2* buf = reinterpret_cast<float2*>(bufs[s]);
    if (chirp_on_load(p.L))  // the manual zap does not depend on the DM: once, on the kept spectrum
      if (int rc = zero_bin_ranges(ctx, buf, p.bins)) return rc;
    for (size_t j = 0; j < n_dm; j++) {
      const detect_out out{0, nullptr, nullptr, d_peaks ? d_peaks + j * p.streams + s : nullptr};
      if (int rc = stream_tail(ctx, p, out, W, buf, h_dms[j], /*phase_table=*/false)) return rc;
      CK(cudaMemcpyAsync(d_sweep + j * p.streams + s, ctx->d_res, sizeof(detect_dev_result), cudaMemcpyDeviceToDevice,
                         ctx->lane.stream));
      if (ev) {  // the trial's series and header, before the next trial overwrites them
        const ev_rows r{ctx->series[0].p, p.L, 0, ctx->d_res, ev_nb, sc.tiles, (unsigned)j, (unsigned)s};
        if (int rc = events_enqueue(ctx, sc, r, 1, sc.count + s, list)) return rc;
      }
    }
  }
  if (ev)
    if (int rc = events_fetch_counts(ctx, sc, list, p.streams)) return rc;
  CK(cudaMemcpyAsync(h_results, d_sweep, n_rec * sizeof(detect_dev_result), cudaMemcpyDeviceToHost, ctx->lane.stream));
  std::vector<detect_dev_peak> own_peaks(outputs && !outputs->h_peaks ? n_rec : 0);
  detect_dev_peak* h_peaks =
      outputs && outputs->h_peaks ? reinterpret_cast<detect_dev_peak*>(outputs->h_peaks) : own_peaks.data();
  if (outputs)
    CK(cudaMemcpyAsync(h_peaks, d_peaks, n_rec * sizeof(detect_dev_peak), cudaMemcpyDeviceToHost, ctx->lane.stream));
  CK(cudaStreamSynchronize(ctx->lane.stream));
  if (ev) events_collect(list, p.streams, *ev);
  if (!outputs) return p.streams;
  int best[4] = {0, 0, 0, 0};
  for (int s = 0; s < p.streams; s++) {
    best[s] = best_trial(h_results, h_peaks, n_dm, p.streams, s);
    if (outputs->h_best_trial) outputs->h_best_trial[s] = best[s];
  }
  if (!outputs->h_series && !user_spec) return p.streams;
  // the best trial once more per stream, from the kept spectrum: its spectrum to d_spectrum[s], its positive series
  // straight from the detector kernel to h_series' row of the stream, its header to h_res[s]
  for (int s = 0; s < p.streams; s++) {
    const detect_out out{0, p.series_row(outputs->h_series, s)};
    float2* dst = user_spec ? reinterpret_cast<float2*>(outputs->d_spectrum[s]) : W;
    CK(cudaMemcpyAsync(ctx->lane.mean, d_means + s, sizeof(float), cudaMemcpyDeviceToDevice, ctx->lane.stream));
    if (int rc = stream_tail(ctx, p, out, dst, reinterpret_cast<float2*>(bufs[s]), h_dms[best[s]], /*phase_table=*/false))
      return rc;
    CK(cudaMemcpyAsync(ctx->h_res + s, ctx->d_res, sizeof(detect_dev_result), cudaMemcpyDeviceToHost, ctx->lane.stream));
  }
  CK(cudaStreamSynchronize(ctx->lane.stream));
  // same kernels on the same input: the re-run must reproduce the loop's header of that trial bit for bit
  for (int s = 0; s < p.streams; s++)
    if (std::memcmp(ctx->h_res + s, h_results + (size_t)best[s] * p.streams + s, sizeof(detect_dev_result)) != 0)
      return fail(ctx, SRTB_B200_E_CUDA,
                  "dm_sweep: the best trial's re-run of stream " + std::to_string(s) + " differs from its trial");
  return p.streams;
}

extern "C" int srtb_b200_process_block_dm_sweep_ex(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg,
                                                   const void* baseband, size_t baseband_bytes, int on_device,
                                                   const float* h_dms, size_t n_dm,
                                                   srtb_b200_detect_result* h_results /* [n_dm][streams] */,
                                                   const srtb_b200_sweep_outputs* outputs /* or NULL */) {
  return dm_sweep(ctx, cfg, baseband, baseband_bytes, on_device, h_dms, n_dm, h_results, outputs, nullptr);
}

extern "C" int srtb_b200_process_block_dm_sweep_events(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg,
                                                       const void* baseband, size_t baseband_bytes, int on_device,
                                                       const float* h_dms, size_t n_dm,
                                                       srtb_b200_detect_result* h_results,
                                                       const srtb_b200_sweep_outputs* outputs,
                                                       srtb_b200_event* h_events, size_t max_events,
                                                       uint64_t* n_events) {
  const ev_request ev{h_events, max_events, n_events};
  return dm_sweep(ctx, cfg, baseband, baseband_bytes, on_device, h_dms, n_dm, h_results, outputs, &ev);
}

// ---- incoherent DM search on one stream's dynamic spectrum (incoherent.cuh): every trial's series in one kernel, then
// the detector's scan and boxcars batched over the trials, the best trial chosen on the host by best_trial().

// the incoherent search's plan of (C, band, dm, trials). The shifts: s[d][c] = llround(K (DM_d - dm) (1/f(c)^2 -
// 1/f_ref^2) sample_rate / (2C)), f_ref = float(freq_low + bandwidth) (the chirp's f_c), f(c) = freq_low + bandwidth
// (c + 0.5) / C, all in double; S+ / S- = max(0, max s) / max(0, -min s). Then the trials sorted by DM (stable) and cut
// greedily into groups of at most INC_GROUP whose spread over every channel is at most INC_SPREAD_MAX (a single trial
// has none), so neighbouring trials share a group whatever order they came in. Returns SRTB_B200_E_INVALID for a shift
// that is not finite, SRTB_B200_E_SIZE for one out of range.
// k[c] of the shifts below: channel c's residual delay per unit DM, in spectrum samples (double; the cut-outs use it too)
static double dispersion_k(size_t C, float freq_low, float bandwidth, float sample_rate, size_t c) {
  constexpr double D = 4.148808e3;
  const double f_ref = (double)(float)(freq_low + bandwidth);
  const double scale = (double)sample_rate / (2.0 * (double)C);
  const double f = (double)freq_low + (double)bandwidth * ((double)c + 0.5) / (double)C;
  return (1.0 / (f * f) - 1.0 / (f_ref * f_ref)) * scale * D;
}

static int incoherent_plan_for(size_t C, float freq_low, float bandwidth, float sample_rate, float dm, const float* dms,
                               size_t n_dm, incoherent_plan* pl) {
  std::vector<int64_t>& sh = pl->shifts;
  sh.assign(n_dm * C, 0);
  int64_t hi = 0, lo = 0;
  for (size_t c = 0; c < C; c++) {
    const double k = dispersion_k(C, freq_low, bandwidth, sample_rate, c);
    for (size_t d = 0; d < n_dm; d++) {
      const double v = ((double)dms[d] - (double)dm) * k;
      if (!std::isfinite(v)) return SRTB_B200_E_INVALID;
      if (std::fabs(v) > 4.0e18) return SRTB_B200_E_SIZE;
      const int64_t s = std::llround(v);
      sh[d * C + c] = s;
      hi = std::max(hi, s);
      lo = std::min(lo, s);
    }
  }
  pl->s_plus = (uint64_t)hi;
  pl->s_minus = (uint64_t)(-lo);
  const int64_t s_minus = -lo;
  std::vector<int>& order = pl->order;
  order.resize(n_dm);
  for (size_t d = 0; d < n_dm; d++) order[d] = (int)d;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return dms[a] < dms[b]; });
  pl->groups.clear();
  pl->gspan.clear();
  pl->spread = 0;
  std::vector<int64_t> gmin(C), gmax(C), nmin(C), nmax(C);
  size_t first = 0;
  while (first < n_dm) {
    for (size_t c = 0; c < C; c++) gmin[c] = gmax[c] = sh[(size_t)order[first] * C + c];
    size_t count = 1;
    while (first + count < n_dm && count < (size_t)INC_GROUP) {
      const size_t d = (size_t)order[first + count];
      bool fits = true;
      for (size_t c = 0; c < C && fits; c++) {
        nmin[c] = std::min(gmin[c], sh[d * C + c]);
        nmax[c] = std::max(gmax[c], sh[d * C + c]);
        fits = nmax[c] - nmin[c] <= INC_SPREAD_MAX;
      }
      if (!fits) break;
      gmin.swap(nmin);
      gmax.swap(nmax);
      count++;
    }
    pl->groups.push_back(make_int2((int)first, (int)count));
    for (size_t c = 0; c < C; c++) {
      pl->gspan.push_back(make_int2((int)(gmin[c] + s_minus), (int)(gmax[c] + s_minus)));
      pl->spread = std::max(pl->spread, (unsigned)(gmax[c] - gmin[c]));
    }
    first += count;
  }
  return 0;
}

extern "C" int srtb_b200_incoherent_shifts(size_t chan_count, float freq_low, float bandwidth, float sample_rate,
                                           float dm, const float* h_dms, size_t n_dm, int64_t* shifts,
                                           uint64_t* s_plus, uint64_t* s_minus) {
  if (chan_count == 0 || !h_dms || n_dm == 0)
    return fail(nullptr, SRTB_B200_E_INVALID, "incoherent_shifts: bad argument");
  incoherent_plan pl;
  if (int rc = incoherent_plan_for(chan_count, freq_low, bandwidth, sample_rate, dm, h_dms, n_dm, &pl))
    return fail(nullptr, rc, "incoherent_shifts: a shift is not finite or out of range");
  if (shifts) std::memcpy(shifts, pl.shifts.data(), pl.shifts.size() * sizeof(int64_t));
  if (s_plus) *s_plus = pl.s_plus;
  if (s_minus) *s_minus = pl.s_minus;
  return 0;
}

extern "C" int srtb_b200_incoherent_groups(size_t chan_count, float freq_low, float bandwidth, float sample_rate,
                                           float dm, const float* h_dms, size_t n_dm, int32_t* order, int32_t* groups,
                                           int32_t* gspan, uint64_t* n_groups, uint32_t* spread) {
  if (chan_count == 0 || !h_dms || n_dm == 0 || !n_groups)
    return fail(nullptr, SRTB_B200_E_INVALID, "incoherent_groups: bad argument");
  incoherent_plan pl;
  if (int rc = incoherent_plan_for(chan_count, freq_low, bandwidth, sample_rate, dm, h_dms, n_dm, &pl))
    return fail(nullptr, rc, "incoherent_groups: a shift is not finite or out of range");
  *n_groups = pl.groups.size();
  if (order) std::memcpy(order, pl.order.data(), pl.order.size() * sizeof(int));
  if (groups) std::memcpy(groups, pl.groups.data(), pl.groups.size() * sizeof(int2));
  if (gspan) std::memcpy(gspan, pl.gspan.data(), pl.gspan.size() * sizeof(int2));
  if (spread) *spread = pl.spread;
  return 0;
}

// the plan of (C, band, dm, trials), cached with the kernel's offsets s + S- in sorted order [C][n_dm]
static int incoherent_tables(srtb_b200_ctx* ctx, size_t C, float freq_low, float bandwidth, float sample_rate,
                             float dm, const float* dms, size_t n_dm) {
  std::vector<double> key = {(double)C, freq_low, bandwidth, sample_rate, dm};
  key.reserve(key.size() + n_dm);  // no reallocating insert: g++ 13 warns falsely on it once this is inlined
  key.insert(key.end(), dms, dms + n_dm);
  if (key == ctx->inc.key) return 0;
  ctx->inc.key.clear();
  const incoherent_plan& pl = ctx->inc.plan;
  if (int rc = incoherent_plan_for(C, freq_low, bandwidth, sample_rate, dm, dms, n_dm, &ctx->inc.plan))
    return fail(ctx, rc, "incoherent_dm_search: a shift is not finite or out of range");
  ctx->inc.off.resize(C * n_dm);
  for (size_t c = 0; c < C; c++)
    for (size_t i = 0; i < n_dm; i++)
      ctx->inc.off[c * n_dm + i] = (int)(pl.shifts[(size_t)pl.order[i] * C + c] + (int64_t)pl.s_minus);
  ctx->inc.uploaded = false;
  ctx->inc.key = std::move(key);
  return 0;
}

// ev (or null): every trial's events, listed by two launches after the detector
static int incoherent_dm_search(srtb_b200_ctx* ctx, const void* d_spectrum, size_t time_count, size_t chan_count,
                                size_t time_reserved_count, float freq_low, float bandwidth, float sample_rate,
                                float dm, const float* h_dms, size_t n_dm, float snr, float channel_threshold,
                                size_t max_boxcar_length, srtb_b200_detect_result* h_results, srtb_b200_peak* h_peaks,
                                int32_t* h_best_trial, float* h_series, const ev_request* ev) {
  API_LOCK(ctx);
  if (!ctx || !d_spectrum || !h_dms || !h_results || n_dm == 0 || time_count == 0 || chan_count == 0 ||
      !ev_request_ok(ev))
    return fail(ctx, SRTB_B200_E_INVALID, "incoherent_dm_search: bad argument");
  if (!aligned8(d_spectrum)) return fail(ctx, SRTB_B200_E_INVALID, "incoherent_dm_search: spectrum not 8-byte aligned");
  if (time_reserved_count >= time_count)
    return fail(ctx, SRTB_B200_E_SIZE, "incoherent_dm_search: time_reserved_count >= time_count");
  if (n_dm > SRTB_B200_INCOHERENT_MAX_DMS)
    return fail(ctx, SRTB_B200_E_SIZE, "incoherent_dm_search: more than SRTB_B200_INCOHERENT_MAX_DMS trials");
  if (time_count > ((size_t)1 << 30))
    return fail(ctx, SRTB_B200_E_SIZE, "incoherent_dm_search: time_count above 2^30");
  CK(cudaSetDevice(ctx->device));
  if (int rc = incoherent_tables(ctx, chan_count, freq_low, bandwidth, sample_rate, dm, h_dms, n_dm)) return rc;
  const size_t ts = time_count - time_reserved_count;
  const incoherent_plan& pl = ctx->inc.plan;
  const uint64_t span = pl.s_plus + pl.s_minus;
  if (span + 2 > ts)
    return fail(ctx, SRTB_B200_E_SIZE, "incoherent_dm_search: T = ts - S+ - S- = " +
                                           std::to_string((long long)ts - (long long)span) + " < 2");
  const size_t T = ts - span;
  const unsigned max_nb = boxcar_ctas(max_boxcar_length, T);
  const size_t n_groups = pl.groups.size();
  // device tables: off [C][n_dm] int, order [n_dm] int, gspan [groups][C] int2, groups [groups] int2
  const size_t off_b = chan_count * n_dm * sizeof(int), order_b = n_dm * sizeof(int);
  const size_t gspan_o = (off_b + order_b + 15) & ~(size_t)15, gspan_b = n_groups * chan_count * sizeof(int2);
  const size_t groups_o = gspan_o + gspan_b, tab_b = groups_o + n_groups * sizeof(int2);
  if (ctx->inc_tab.bytes < tab_b) ctx->inc.uploaded = false;
  if (int rc = grow(ctx, ctx->inc_tab, tab_b)) return rc;
  // work: series [n_dm][max_nb][T], scans [n_dm][T], headers [n_dm], peaks [n_dm], tickets [n_dm]
  const size_t series_stride = (size_t)max_nb * T;
  const size_t series_b = n_dm * series_stride * sizeof(float), acc_b = n_dm * T * sizeof(float);
  const size_t res_o = (series_b + acc_b + 255) & ~(size_t)255;
  const size_t peak_o = res_o + n_dm * sizeof(detect_dev_result);
  const size_t ticket_o = peak_o + n_dm * sizeof(detect_dev_peak);
  const size_t work_b = ticket_o + n_dm * sizeof(unsigned);
  if (int rc = grow(ctx, ctx->inc_work, work_b)) return rc;
  ev_scratch sc{};
  ev_list list;
  if (ev)
    if (int rc = events_prepare(ctx, "incoherent_dm_search", n_dm, max_nb, T, 1, ev->max_events, 0, &sc, &list))
      return rc;
  char* tab = ctx->inc_tab.p;
  char* work = ctx->inc_work.p;
  float* d_series = reinterpret_cast<float*>(work);
  float* d_acc = reinterpret_cast<float*>(work + series_b);
  detect_dev_result* d_res = reinterpret_cast<detect_dev_result*>(work + res_o);
  detect_dev_peak* d_peak = reinterpret_cast<detect_dev_peak*>(work + peak_o);
  unsigned* d_ticket = reinterpret_cast<unsigned*>(work + ticket_o);
  cudaStream_t st = ctx->lane.stream;
  if (!ctx->inc.uploaded) {  // the host vectors live in the ctx, so the copies may complete after we return
    CK(cudaMemcpyAsync(tab, ctx->inc.off.data(), off_b, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(tab + off_b, pl.order.data(), order_b, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(tab + gspan_o, pl.gspan.data(), gspan_b, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(tab + groups_o, pl.groups.data(), n_groups * sizeof(int2), cudaMemcpyHostToDevice, st));
    ctx->inc.uploaded = true;
  }
  CK(cudaMemsetAsync(work + res_o, 0, work_b - res_o, st));  // headers (zero_count is atomically added), peaks, tickets
  const unsigned spread = pl.spread;
  const size_t smem = incoherent_smem_bytes(spread);
  if (smem > 48 * 1024)  // once, for the largest spread any group may have
    if (int rc = set_smem_max(ctx, incoherent_dedisperse_kernel, incoherent_smem_bytes(INC_SPREAD_MAX))) return rc;
  // gridDim.y is at most 65535: a longer series (T above 65535 INC_TILE, just over 2^24) has CTAs form several tiles
  const dim3 grid((unsigned)n_groups, (unsigned)std::min<size_t>((T + INC_TILE - 1) / INC_TILE, 65535));
  CK(launch(ctx, false, incoherent_dedisperse_kernel, grid, INC_THREADS, smem, static_cast<const float2*>(d_spectrum),
            time_count, chan_count, T, n_dm, reinterpret_cast<const int*>(tab),
            reinterpret_cast<const int2*>(tab + gspan_o), reinterpret_cast<const int2*>(tab + groups_o),
            reinterpret_cast<const int*>(tab + off_b), INC_TILE + spread, d_series, series_stride));
  // the series are already in place: no partial sums (partial == nullptr); one CTA per trial zero-counts and scans
  CK(launch(ctx, false, colsum_final_scan_kernel, dim3(1, (unsigned)n_dm), 1024, 0, nullptr, T, 0, d_series, d_acc,
            static_cast<const float2*>(d_spectrum), time_count, chan_count, channel_threshold, max_boxcar_length,
            d_ticket, d_res, series_stride, T, nullptr));
  CK(launch(ctx, false, detect_boxcar_kernel<true>, dim3(max_nb, (unsigned)n_dm), 1024, 0, d_series, T, d_acc, T, snr,
            d_res, nullptr, d_peak, series_stride, T));
  if (ev) {
    const ev_rows r{d_series, T, series_stride, d_res, max_nb, sc.tiles, 0u, 0u};
    if (int rc = events_enqueue(ctx, sc, r, n_dm, sc.count, list)) return rc;
    if (int rc = events_fetch_counts(ctx, sc, list, 1)) return rc;
  }
  std::vector<srtb_b200_peak> own_peaks(h_peaks ? 0 : n_dm);
  srtb_b200_peak* peaks = h_peaks ? h_peaks : own_peaks.data();
  CK(cudaMemcpyAsync(h_results, d_res, n_dm * sizeof(detect_dev_result), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(peaks, d_peak, n_dm * sizeof(detect_dev_peak), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (ev) events_collect(list, 1, *ev);
  const int best = best_trial(h_results, reinterpret_cast<const detect_dev_peak*>(peaks), n_dm, 1, 0);
  if (h_best_trial) *h_best_trial = best;
  if (!h_series) return 0;
  // the best trial's positive series, rows of T floats as process_block writes them (only the positive rows)
  const srtb_b200_detect_result& r = h_results[best];
  bool any = false;
  for (int b = 0; b < r.n_boxcars; b++) {
    if (r.signal_count[b] == 0) continue;
    CK(cudaMemcpyAsync(h_series + (size_t)b * T, d_series + (size_t)best * series_stride + (size_t)b * T,
                       r.series_length[b] * sizeof(float), cudaMemcpyDeviceToHost, st));
    any = true;
  }
  if (any) CK(cudaStreamSynchronize(st));
  return 0;
}

extern "C" int srtb_b200_incoherent_dm_search(srtb_b200_ctx* ctx, const void* d_spectrum, size_t time_count,
                                              size_t chan_count, size_t time_reserved_count, float freq_low,
                                              float bandwidth, float sample_rate, float dm, const float* h_dms,
                                              size_t n_dm, float snr, float channel_threshold,
                                              size_t max_boxcar_length, srtb_b200_detect_result* h_results,
                                              srtb_b200_peak* h_peaks, int32_t* h_best_trial, float* h_series) {
  return incoherent_dm_search(ctx, d_spectrum, time_count, chan_count, time_reserved_count, freq_low, bandwidth,
                              sample_rate, dm, h_dms, n_dm, snr, channel_threshold, max_boxcar_length, h_results,
                              h_peaks, h_best_trial, h_series, nullptr);
}

extern "C" int srtb_b200_incoherent_dm_search_events(srtb_b200_ctx* ctx, const void* d_spectrum, size_t time_count,
                                                     size_t chan_count, size_t time_reserved_count, float freq_low,
                                                     float bandwidth, float sample_rate, float dm, const float* h_dms,
                                                     size_t n_dm, float snr, float channel_threshold,
                                                     size_t max_boxcar_length, srtb_b200_detect_result* h_results,
                                                     srtb_b200_peak* h_peaks, int32_t* h_best_trial, float* h_series,
                                                     srtb_b200_event* h_events, size_t max_events, uint64_t* n_events) {
  const ev_request ev{h_events, max_events, n_events};
  return incoherent_dm_search(ctx, d_spectrum, time_count, chan_count, time_reserved_count, freq_low, bandwidth,
                              sample_rate, dm, h_dms, n_dm, snr, channel_threshold, max_boxcar_length, h_results,
                              h_peaks, h_best_trial, h_series, &ev);
}

// ---- candidate cut-outs (cutout.cuh): the frequency-time image and DM-time plane of every request in four launches.

// the scratch of one call, each part 256-byte aligned: k [C] double, requests [n], row DMs [n][n_rows], bases and image
// offsets [n][C], group spans [n][groups][C], decimated power [n][C][Wd], then the images ft [n][nsub][W] and dmt
// [n][n_rows][W]
struct cutout_layout {
  size_t k, req, row_dms, base, ft_off, gspan, d, ft, dmt, bytes;
  cutout_layout(size_t n, size_t C, size_t Wd, size_t W, size_t nsub, size_t n_rows, size_t groups) {
    size_t o = 0;
    auto take = [&](size_t b) {
      const size_t at = o;
      o += (b + 255) & ~(size_t)255;
      return at;
    };
    k = take(C * sizeof(double));
    req = take(n * sizeof(cut_request));
    row_dms = take(n * n_rows * sizeof(float));
    base = take(n * C * sizeof(int));
    ft_off = take(n * C * sizeof(int));
    gspan = take(n * groups * C * sizeof(int2));
    d = take(n * C * Wd * sizeof(float));
    ft = take(n * nsub * W * sizeof(float));
    dmt = take(n * n_rows * W * sizeof(float));
    bytes = o;
  }
};

// an upper bound of |llround(a) - llround(b)| over the shifts of two DMs lo, hi in any channel, k_max = max |k[c]|: the
// difference of the real shifts plus one for the rounding, with room for their float64 and float32 rounding errors
static double cutout_shift_bound(float lo, float hi, double k_max, unsigned q) {
  const double d = std::fabs((double)hi - (double)lo) + std::ldexp(std::fabs((double)hi) + std::fabs((double)lo), -20);
  return std::floor(d * k_max / (double)q * (1.0 + 1e-9)) + 2.0;
}

extern "C" int srtb_b200_candidate_cutouts(srtb_b200_ctx* ctx, const void* const* d_spectra, int streams,
                                           size_t time_count, size_t chan_count, size_t time_reserved_count,
                                           float freq_low, float bandwidth, float sample_rate, float dm,
                                           const srtb_b200_cutout_request* h_requests, size_t n, size_t width,
                                           size_t nsub, size_t n_rows, float* h_ft, float* h_dmt, float* h_row_dms) {
  API_LOCK(ctx);
  const std::string who = "candidate_cutouts: ";
  if (!ctx || !d_spectra || !h_requests || !h_ft || !h_dmt || time_count == 0 || chan_count == 0)
    return fail(ctx, SRTB_B200_E_INVALID, who + "bad argument");
  if (streams < 1 || streams > 4) return fail(ctx, SRTB_B200_E_INVALID, who + "streams must be 1 to 4");
  for (int s = 0; s < streams; s++) {
    if (!d_spectra[s]) return fail(ctx, SRTB_B200_E_INVALID, who + "a spectrum is null");
    if (!aligned8(d_spectra[s])) return fail(ctx, SRTB_B200_E_INVALID, who + "a spectrum is not 8-byte aligned");
  }
  if (n == 0) return fail(ctx, SRTB_B200_E_INVALID, who + "no requests");
  if (n > 65535) return fail(ctx, SRTB_B200_E_SIZE, who + "more than 65535 requests");
  if (width % 2) return fail(ctx, SRTB_B200_E_INVALID, who + "width must be even");
  if (width < 2 || width > 4096) return fail(ctx, SRTB_B200_E_SIZE, who + "width outside 2 .. 4096");
  if (n_rows < 1 || n_rows > 4096) return fail(ctx, SRTB_B200_E_SIZE, who + "n_rows outside 1 .. 4096");
  if (nsub == 0 || chan_count % nsub) return fail(ctx, SRTB_B200_E_INVALID, who + "nsub must divide chan_count");
  if (!std::isfinite(dm)) return fail(ctx, SRTB_B200_E_INVALID, who + "dm is not finite");
  for (size_t i = 0; i < n; i++) {
    const srtb_b200_cutout_request& r = h_requests[i];
    if (r.decimation == 0) return fail(ctx, SRTB_B200_E_INVALID, who + "a decimation is 0");
    if (r.decimation > (1u << 20)) return fail(ctx, SRTB_B200_E_SIZE, who + "a decimation above 2^20");
    if (!std::isfinite(r.dm) || !std::isfinite(r.dm_halfwidth))
      return fail(ctx, SRTB_B200_E_INVALID, who + "a request's dm or dm_halfwidth is not finite");
  }
  if (time_reserved_count >= time_count)
    return fail(ctx, SRTB_B200_E_SIZE, who + "time_reserved_count >= time_count");
  const size_t C = chan_count, W = width, R = n_rows;
  std::vector<double> k(C);
  double k_max = 0;
  for (size_t c = 0; c < C; c++) {
    k[c] = dispersion_k(C, freq_low, bandwidth, sample_rate, c);
    if (!std::isfinite(k[c])) return fail(ctx, SRTB_B200_E_INVALID, who + "a shift is not finite");
    k_max = std::max(k_max, std::fabs(k[c]));
  }
  // every shift fits 2^24 decimated bins and every sample index int64 (|center| < 2^62): each request's row DMs span
  // [first, last] (monotone in the row), its own DM among them. The window of decimated bins is W + the widest span
  // of one channel's shifts; groups of rows_per_group rows spread at most INC_SPREAD_MAX bins in any channel
  std::vector<cut_request> req(n);
  double wspan = 0;
  for (size_t i = 0; i < n; i++) {
    const srtb_b200_cutout_request& r = h_requests[i];
    const float first = cut_row_dm(r.dm, r.dm_halfwidth, 0, (unsigned)R);
    const float last = cut_row_dm(r.dm, r.dm_halfwidth, (unsigned)R - 1, (unsigned)R);
    for (float d : {first, last, r.dm}) {
      const double v = ((double)d - (double)dm) * k_max / (double)r.decimation;
      if (!std::isfinite(v)) return fail(ctx, SRTB_B200_E_INVALID, who + "a shift is not finite");
      if (std::fabs(v) > (double)(1 << 24)) return fail(ctx, SRTB_B200_E_SIZE, who + "a shift out of range (2^24 bins)");
    }
    if (r.center >= ((int64_t)1 << 62) || r.center <= -((int64_t)1 << 62))
      return fail(ctx, SRTB_B200_E_SIZE, who + "a center out of range (2^62)");
    wspan = std::max(wspan, cutout_shift_bound(first, last, k_max, r.decimation));
    req[i] = cut_request{(long long)r.center - (long long)(W / 2) * (long long)r.decimation, r.decimation, r.dm,
                         r.dm_halfwidth};
  }
  unsigned rows_per_group = INC_GROUP;
  for (;; rows_per_group /= 2) {
    bool fits = true;
    for (size_t i = 0; i < n && fits && rows_per_group > 1; i++) {
      const srtb_b200_cutout_request& r = h_requests[i];
      for (size_t r0 = 0; r0 < R && fits; r0 += rows_per_group) {
        const size_t r1 = std::min(r0 + rows_per_group, R) - 1;
        fits = cutout_shift_bound(cut_row_dm(r.dm, r.dm_halfwidth, (unsigned)r0, (unsigned)R),
                                  cut_row_dm(r.dm, r.dm_halfwidth, (unsigned)r1, (unsigned)R), k_max,
                                  r.decimation) <= INC_SPREAD_MAX;
      }
    }
    if (fits) break;
  }
  const unsigned groups = (unsigned)((R + rows_per_group - 1) / rows_per_group);
  const unsigned spread = rows_per_group > 1 ? INC_SPREAD_MAX : 0;
  const size_t Wd = W + (size_t)wspan;
  const unsigned d_tiles = (unsigned)((Wd + CUT_THREADS - 1) / CUT_THREADS);
  const unsigned w_tiles = (unsigned)((W + CUT_THREADS - 1) / CUT_THREADS);
  const unsigned p_tiles = (unsigned)((W + INC_TILE - 1) / INC_TILE);
  if ((double)C * d_tiles > 2147483647.0 || (double)nsub * w_tiles > 2147483647.0)
    return fail(ctx, SRTB_B200_E_SIZE, who + "a shift out of range (grid)");
  CK(cudaSetDevice(ctx->device));
  const cutout_layout lay(n, C, Wd, W, nsub, R, groups);
  if (int rc = grow(ctx, ctx->cut_work, lay.bytes)) return rc;
  char* w = ctx->cut_work.p;
  cudaStream_t st = ctx->lane.stream;
  // pageable sources: each copy returns once its bytes are staged, so the host vectors may go when we return
  CK(cudaMemcpyAsync(w + lay.k, k.data(), C * sizeof(double), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(w + lay.req, req.data(), n * sizeof(cut_request), cudaMemcpyHostToDevice, st));
  const auto* d_req = reinterpret_cast<const cut_request*>(w + lay.req);
  const auto* d_k = reinterpret_cast<const double*>(w + lay.k);
  auto* d_row_dms = reinterpret_cast<float*>(w + lay.row_dms);
  auto* d_base = reinterpret_cast<int*>(w + lay.base);
  auto* d_ft_off = reinterpret_cast<int*>(w + lay.ft_off);
  auto* d_gspan = reinterpret_cast<int2*>(w + lay.gspan);
  auto* d_D = reinterpret_cast<float*>(w + lay.d);
  auto* d_ft = reinterpret_cast<float*>(w + lay.ft);
  auto* d_dmt = reinterpret_cast<float*>(w + lay.dmt);
  cut_spectra sp{};
  for (int s = 0; s < streams; s++) sp.x[s] = static_cast<const float2*>(d_spectra[s]);
  sp.streams = streams;
  sp.L = time_count;
  sp.C = C;
  sp.ts = time_count - time_reserved_count;
  const unsigned plan_x = (unsigned)((std::max(C, R) + CUT_THREADS - 1) / CUT_THREADS);
  CK(launch(ctx, false, cutout_plan_kernel, dim3(plan_x, (unsigned)n), CUT_THREADS, 0, d_req, d_k, C, (double)dm,
            (unsigned)R, rows_per_group, groups, d_row_dms, d_base, d_ft_off, d_gspan));
  CK(launch(ctx, false, cutout_decimate_kernel, dim3((unsigned)(C * d_tiles), (unsigned)n), CUT_THREADS, 0, sp, d_req,
            static_cast<const int*>(d_base), Wd, d_tiles, d_D));
  CK(launch(ctx, false, cutout_ft_kernel, dim3((unsigned)(nsub * w_tiles), (unsigned)n), CUT_THREADS, 0,
            static_cast<const float*>(d_D), static_cast<const int*>(d_ft_off), C, Wd, (unsigned)W, (unsigned)nsub,
            w_tiles, d_ft));
  CK(launch(ctx, false, cutout_plane_kernel, dim3(groups * p_tiles, (unsigned)n), INC_THREADS,
            cutout_plane_smem_bytes(spread), static_cast<const float*>(d_D), C, Wd,
            static_cast<const int2*>(d_gspan), static_cast<const int*>(d_base), d_k,
            static_cast<const float*>(d_row_dms), d_req, (double)dm, (unsigned)R, rows_per_group, groups,
            (unsigned)W, (unsigned)(INC_TILE + spread), d_dmt));
  CK(cudaMemcpyAsync(h_ft, d_ft, n * nsub * W * sizeof(float), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(h_dmt, d_dmt, n * R * W * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (h_row_dms) CK(cudaMemcpyAsync(h_row_dms, d_row_dms, n * R * sizeof(float), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return 0;
}

// ---- fold at a pulsar period (fold.cuh): the bin plan of each time tile, one read of the spectra into per-CTA bin
// rows, and the rows' sum in a fixed order.

extern "C" int srtb_b200_fold_phase(double period, double period_derivative, double sample_rate,
                                    uint64_t samples_per_spectrum_sample, uint64_t first_sample, double* phi0,
                                    double* a, double* b) {
  if (!phi0 || !a || !b || samples_per_spectrum_sample == 0)
    return fail(nullptr, SRTB_B200_E_INVALID, "fold_phase: bad argument");
  if (!std::isfinite(period) || !(period > 0) || !std::isfinite(period_derivative) || !std::isfinite(sample_rate) ||
      !(sample_rate > 0))
    return fail(nullptr, SRTB_B200_E_INVALID, "fold_phase: period and sample_rate must be finite and positive, "
                                              "period_derivative finite");
  // the order of every operation is part of the definition (include/srtb_b200.h)
  const double t0 = (double)first_sample / sample_rate;
  const double q = period_derivative / (period * period);
  const double phi = t0 / period - (0.5 * q) * (t0 * t0);
  const double delta = (double)samples_per_spectrum_sample / sample_rate;
  *phi0 = phi - std::floor(phi);
  *a = (1.0 / period - q * t0) * delta;
  *b = (-0.5 * q) * (delta * delta);
  return 0;
}

// srtb_b200_fold and srtb_b200_fold_coherence past their own pointer checks: the checks both make (messages prefixed
// `who`), then the bin plan, `kern` (its leading arguments `in`), the rows' sum and the copies back. kern's CTAs take G
// channels of one of S streams by R tile ranges, up to one wave of per_sm CTAs per SM; a subband has P output rows (the
// streams, or the four coherence products), and the first S nsub kept counts are copied back.
template <class... KArgs, class... In>
static int fold_run(srtb_b200_ctx* ctx, const char* who, size_t time_count, size_t chan_count, size_t fold_count,
                    double phi0, double a, double b, size_t nbin, size_t nsub, double* h_out, uint64_t* h_hits,
                    uint32_t* h_kept, size_t P, size_t S, size_t per_sm, void (*kern)(KArgs...), int threads,
                    size_t (*smem_bytes)(int), In... in) {
  const std::string pre = std::string(who) + ": ";
  if (fold_count == 0 || fold_count > time_count)
    return fail(ctx, SRTB_B200_E_SIZE, pre + "fold_count must be 1 to time_count");
  if (nbin < 1 || nbin > (size_t)FOLD_MAX_BINS) return fail(ctx, SRTB_B200_E_SIZE, pre + "nbin must be 1 to 4096");
  if (nsub == 0 || chan_count % nsub) return fail(ctx, SRTB_B200_E_SIZE, pre + "nsub must divide chan_count");
  if (chan_count > ((size_t)1 << 24) || fold_count > ((size_t)1 << 40))
    return fail(ctx, SRTB_B200_E_SIZE, pre + "chan_count above 2^24 or fold_count above 2^40");
  if (!std::isfinite(phi0) || !std::isfinite(a) || !std::isfinite(b))
    return fail(ctx, SRTB_B200_E_INVALID, pre + "a phase coefficient is not finite");
  CK(cudaSetDevice(ctx->device));
  const size_t C = chan_count, csub = C / nsub;
  size_t G = std::min<size_t>(csub, FOLD_MAX_GROUP);
  while (csub % G) G--;  // channels per CTA: the largest divisor of the subband width up to FOLD_MAX_GROUP
  const size_t ntiles = (fold_count + FOLD_TILE - 1) / FOLD_TILE, ctas = S * (C / G);
  // tile ranges per channel group: up to one wave of the CTAs an SM holds (nsub = 1 then still spreads over the SMs)
  const size_t target = (size_t)ctx->sm_count * per_sm;
  const size_t R = std::max<size_t>(1, std::min<size_t>(ntiles, target / ctas));
  const size_t gps = csub / G, rows_per_output = gps * R, outputs = P * nsub * nbin;
  // scratch: plan u32 [ntiles][FOLD_TILE], hits u64 [nbin], profile f64 [P][nsub][nbin], kept u32 [P][nsub] (for the
  // coherence products the same count four times: fold_finish_kernel's layout); with more than one CTA row per output
  // also rows f64 [P (C / G) R nbin] and kept rows u32 [P (C / G)]
  const auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
  const size_t hits_o = up(ntiles * FOLD_TILE * sizeof(uint32_t));
  const size_t prof_o = hits_o + up(nbin * sizeof(uint64_t));
  const size_t kept_o = prof_o + up(outputs * sizeof(double));
  const size_t rows_o = kept_o + up(P * nsub * sizeof(uint32_t));
  const bool finish = rows_per_output > 1;
  const size_t krow_o = rows_o + (finish ? up(P * (C / G) * R * nbin * sizeof(double)) : 0);
  const size_t work_b = krow_o + (finish ? P * (C / G) * sizeof(uint32_t) : 0);
  if (int rc = grow(ctx, ctx->fold_work, work_b)) return rc;
  char* w = ctx->fold_work.p;
  uint32_t* d_plan = reinterpret_cast<uint32_t*>(w);
  unsigned long long* d_hits = reinterpret_cast<unsigned long long*>(w + hits_o);
  double* d_prof = reinterpret_cast<double*>(w + prof_o);
  unsigned* d_kept = reinterpret_cast<unsigned*>(w + kept_o);
  double* d_rows = finish ? reinterpret_cast<double*>(w + rows_o) : d_prof;
  unsigned* d_krows = finish ? reinterpret_cast<unsigned*>(w + krow_o) : d_kept;
  cudaStream_t st = ctx->lane.stream;
  if (int rc = set_smem_max(ctx, kern, smem_bytes(FOLD_MAX_BINS))) return rc;
  CK(cudaMemsetAsync(d_hits, 0, nbin * sizeof(uint64_t), st));
  CK(launch(ctx, false, fold_plan_kernel, (unsigned)ntiles, FOLD_PLAN_THREADS, 0, phi0, a, b, (int)nbin,
            (long long)fold_count, d_plan, d_hits));
  CK(launch(ctx, false, kern, dim3((unsigned)ctas, (unsigned)R), threads, smem_bytes((int)nbin), in..., time_count,
            (int)C, (int)G, (int)nbin, (long long)fold_count, (int)ntiles, d_plan, d_rows, d_krows));
  if (finish)
    CK(launch(ctx, false, fold_finish_kernel, (unsigned)((outputs + 255) / 256), 256, 0, d_rows, d_krows,
              (int)rows_per_output, (int)gps, (int)nbin, outputs, d_prof, d_kept));
  CK(cudaMemcpyAsync(h_out, d_prof, outputs * sizeof(double), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(h_hits, d_hits, nbin * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(h_kept, d_kept, S * nsub * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return 0;
}

extern "C" int srtb_b200_fold(srtb_b200_ctx* ctx, const void* const* d_spectra, int streams, size_t time_count,
                              size_t chan_count, size_t fold_count, double phi0, double a, double b, size_t nbin,
                              size_t nsub, double* h_profile, uint64_t* h_hits, uint32_t* h_kept) {
  API_LOCK(ctx);
  if (!ctx || !d_spectra || !h_profile || !h_hits || !h_kept || time_count == 0 || chan_count == 0)
    return fail(ctx, SRTB_B200_E_INVALID, "fold: bad argument");
  if (streams < 1 || streams > 4) return fail(ctx, SRTB_B200_E_INVALID, "fold: streams must be 1 to 4");
  fold_spectra sp{};
  for (int s = 0; s < streams; s++) {
    if (!d_spectra[s]) return fail(ctx, SRTB_B200_E_INVALID, "fold: spectrum " + std::to_string(s) + " is null");
    if (!aligned8(d_spectra[s]))
      return fail(ctx, SRTB_B200_E_INVALID, "fold: spectrum " + std::to_string(s) + " is not 8-byte aligned");
    sp.x[s] = static_cast<const float2*>(d_spectra[s]);
  }
  // four CTAs per SM (fold_kernel's launch bounds)
  return fold_run(ctx, "fold", time_count, chan_count, fold_count, phi0, a, b, nbin, nsub, h_profile, h_hits, h_kept,
                  streams, streams, 4, fold_kernel, FOLD_THREADS, fold_smem_bytes, sp);
}

// the coherence products of a stream pair: srtb_b200_fold's plan and finish around fold_coherence_kernel, whose CTAs
// read both streams and whose CTA rows stand for four streams (AA, BB, CR, CI)
extern "C" int srtb_b200_fold_coherence(srtb_b200_ctx* ctx, const void* d_x, const void* d_y, size_t time_count,
                                        size_t chan_count, size_t fold_count, double phi0, double a, double b,
                                        size_t nbin, size_t nsub, double* h_coherence, uint64_t* h_hits,
                                        uint32_t* h_kept) {
  API_LOCK(ctx);
  if (!ctx || !d_x || !d_y || !h_coherence || !h_hits || !h_kept || time_count == 0 || chan_count == 0)
    return fail(ctx, SRTB_B200_E_INVALID, "fold_coherence: bad argument");
  if (!aligned8(d_x) || !aligned8(d_y))
    return fail(ctx, SRTB_B200_E_INVALID, "fold_coherence: a spectrum is not 8-byte aligned");
  if (d_x == d_y) return fail(ctx, SRTB_B200_E_INVALID, "fold_coherence: d_x and d_y are the same spectrum");
  // two CTAs per SM (the shared memory of nbin <= 1024 allows two); the four products share one kept count
  return fold_run(ctx, "fold_coherence", time_count, chan_count, fold_count, phi0, a, b, nbin, nsub, h_coherence,
                  h_hits, h_kept, 4, 1, 2, fold_coherence_kernel, FOLD_COH_THREADS, fold_coherence_smem_bytes,
                  static_cast<const float2*>(d_x), static_cast<const float2*>(d_y));
}

// tickets wrap at a multiple of the slot count, so ticket % SRTB_B200_RING_SLOTS is always the slot that was used
static inline int ring_ticket(uint64_t submit_count) {
  return (int)(submit_count % ((uint64_t)SRTB_B200_RING_SLOTS << 28));
}
extern "C" int srtb_b200_debug_set_submit_count(srtb_b200_ctx* ctx, uint64_t value) {
  API_LOCK(ctx);
  if (!ctx) return fail(nullptr, SRTB_B200_E_INVALID, "debug_set_submit_count: ctx is null");
  for (const ring_slot& rs : ctx->ring)
    if (rs.busy) return fail(ctx, SRTB_B200_E_INVALID, "debug_set_submit_count: ring not empty");
  ctx->submit_count = value;
  return 0;
}

// ---- pipelined ingest: the pinned-host ring of SURVEY section 8e -------------------------------
// submit() copies block k on a dedicated copy stream while block k-1 computes; collect() waits for
// one block's results. Up to SRTB_B200_RING_SLOTS blocks may be in flight.
// max_events (or null: the plain entry): list every detector's events into the slot's pinned list
static int submit_ring(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg, const void* baseband,
                       size_t baseband_bytes, int on_device, const srtb_b200_block_outputs* outputs,
                       const size_t* max_events) {
  API_LOCK(ctx);
  if (!ctx || !cfg || !baseband) return fail(ctx, SRTB_B200_E_INVALID, "submit_block: null argument");
  if (max_events && *max_events > ((size_t)1 << 32))
    return fail(ctx, SRTB_B200_E_INVALID, "submit_block_events: max_events above 2^32");
  CK(cudaSetDevice(ctx->device));
  const int k = (int)(ctx->submit_count % SRTB_B200_RING_SLOTS);
  ring_slot& rs = ctx->ring[k];
  if (rs.busy) return fail(ctx, SRTB_B200_E_INVALID, "submit_block: ring full, collect a block first");
  block_params p;
  if (int rc = block_params_for(ctx, cfg, "process_block", &p)) return rc;
  if (!rs.done)
    for (ring_slot& r : ctx->ring)
      if (!r.done) CK(cudaEventCreateWithFlags(&r.done, cudaEventDisableTiming));
  // outputs: the caller's buffers (the work's own buffer, as in the reference) or this slot's ctx-owned ones
  float* bufs[4] = {nullptr, nullptr, nullptr, nullptr};
  bool user_spec = false;
  if (int rc = caller_spectra(ctx, "submit_block", outputs ? outputs->d_spectrum : nullptr, p.streams, &user_spec))
    return rc;
  if (user_spec) {
    for (int s = 0; s < p.streams; s++) bufs[s] = outputs->d_spectrum[s];
  } else if (int rc = own_stream_bufs(ctx, p, rs.stream_buf, bufs)) {
    return rc;
  }
  const size_t rows = (size_t)p.streams + (cfg->signal_detect_sum_streams ? 1 : 0);  // of the series and the events
  float* h_series = outputs ? outputs->h_series : nullptr;
  if (!h_series) {
    if (int rc = grow(ctx, rs.h_series, rows * SRTB_B200_MAX_BOXCARS * p.L * sizeof(float))) return rc;
    h_series = rs.h_series.p;
  }
  const void* d_baseband = baseband;
  if (!on_device) {
    if (!ctx->copy_stream) {
      CK(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
      for (ring_slot& r : ctx->ring) CK(cudaEventCreateWithFlags(&r.h2d, cudaEventDisableTiming));
    }
    if (int rc = grow(ctx, rs.baseband, baseband_bytes)) return rc;
    CK(cudaMemcpyAsync(rs.baseband.p, baseband, baseband_bytes, cudaMemcpyHostToDevice, ctx->copy_stream));
    CK(cudaEventRecord(rs.h2d, ctx->copy_stream));
    CK(cudaStreamWaitEvent(ctx->lane.stream, rs.h2d, 0));
    d_baseband = rs.baseband.p;
  }
  ev_list list;
  if (max_events)
    if (int rc = ev_list_for(ctx, rs.ev, rows, *max_events, &list)) return rc;
  bool alt_used = false;
  if (int rc = block_enqueue(ctx, p, d_baseband, baseband_bytes, RES_GROUP * (1 + k), bufs, h_series, /*join_lanes=*/false,
                             &alt_used, max_events ? &list : nullptr))
    return rc;
  rs.list = list;
  rs.streams = p.streams;
  rs.sum = cfg->signal_detect_sum_streams != 0;
  CK(cudaEventRecord(rs.done, ctx->lane.stream));
  rs.alt_used = alt_used;
  if (alt_used) {
    if (!rs.done_alt) CK(cudaEventCreateWithFlags(&rs.done_alt, cudaEventDisableTiming));
    CK(cudaEventRecord(rs.done_alt, ctx->alt.stream));
  }
  for (int s = 0; s < 4; s++) rs.out_spectrum[s] = bufs[s];
  rs.out_series = h_series;
  rs.busy = true;
  const int ticket = ring_ticket(ctx->submit_count);
  rs.ticket = ticket;
  ctx->submit_count++;
  return ticket;
}

extern "C" int srtb_b200_submit_block_ex(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg, const void* baseband,
                                         size_t baseband_bytes, int on_device, const srtb_b200_block_outputs* outputs) {
  return submit_ring(ctx, cfg, baseband, baseband_bytes, on_device, outputs, nullptr);
}

extern "C" int srtb_b200_submit_block_events(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg,
                                             const void* baseband, size_t baseband_bytes, int on_device,
                                             const srtb_b200_block_outputs* outputs, size_t max_events) {
  return submit_ring(ctx, cfg, baseband, baseband_bytes, on_device, outputs, &max_events);
}

extern "C" int srtb_b200_submit_block(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg,
                                      const void* h_baseband, size_t baseband_bytes) {
  return srtb_b200_submit_block_ex(ctx, cfg, h_baseband, baseband_bytes, 0, nullptr);
}

// same ring, input already on the device (no copy): lets a device-resident producer keep the GPU fed
extern "C" int srtb_b200_submit_block_device(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg,
                                             const void* d_baseband, size_t baseband_bytes) {
  return srtb_b200_submit_block_ex(ctx, cfg, d_baseband, baseband_bytes, 1, nullptr);
}

// events (or false: the plain entry): the slot's event list and counts to h_events / n_events
static int collect_ring(srtb_b200_ctx* ctx, int ticket, srtb_b200_detect_result* h_results, const float** h_series,
                        const void** d_spectrum, bool events, const srtb_b200_event** h_events, uint64_t* n_events) {
  API_LOCK(ctx);
  if (!ctx || !h_results || ticket < 0 || (events && !n_events))
    return fail(ctx, SRTB_B200_E_INVALID, "collect_block: bad argument");
  const int k = ticket % SRTB_B200_RING_SLOTS;
  ring_slot& rs = ctx->ring[k];
  if (!rs.busy || rs.ticket != ticket)
    return fail(ctx, SRTB_B200_E_INVALID, "collect_block: nothing submitted under this ticket");
  if (events && !rs.list.p)
    return fail(ctx, SRTB_B200_E_INVALID, "collect_block_events: the block was not submitted with submit_block_events");
  if (events && !h_events && rs.list.max_events > 0)
    return fail(ctx, SRTB_B200_E_INVALID, "collect_block_events: h_events is null and the block lists events");
  CK(cudaSetDevice(ctx->device));
  {
    const cudaEvent_t e0 = rs.done, e1 = rs.alt_used ? rs.done_alt : nullptr;
    api_lock_.unlock();  // the wait runs unlocked (a ticket is collected once, by one thread)
    CK(cudaEventSynchronize(e0));
    if (e1) CK(cudaEventSynchronize(e1));
    api_lock_.lock();
  }
  const int streams = rs.streams;
  const detect_dev_result* res = ctx->h_res + RES_GROUP * (1 + k);
  std::memcpy(h_results, res, sizeof(srtb_b200_detect_result) * streams);
  if (rs.sum) std::memcpy(h_results + streams, res + SUM_SLOT, sizeof(srtb_b200_detect_result));
  if (h_series) *h_series = rs.out_series;
  if (d_spectrum)
    for (int s = 0; s < 4; s++) d_spectrum[s] = s < streams ? rs.out_spectrum[s] : nullptr;
  if (events) {
    for (int r = 0; r < streams + (rs.sum ? 1 : 0); r++) n_events[r] = rs.list.counts()[r];
    if (h_events) *h_events = reinterpret_cast<const srtb_b200_event*>(rs.list.row(0));
  }
  rs.busy = false;
  return streams;
}

extern "C" int srtb_b200_collect_block_ex(srtb_b200_ctx* ctx, int ticket, srtb_b200_detect_result* h_results,
                                          const float** h_series, const void** d_spectrum) {
  return collect_ring(ctx, ticket, h_results, h_series, d_spectrum, false, nullptr, nullptr);
}

extern "C" int srtb_b200_collect_block_events(srtb_b200_ctx* ctx, int ticket, srtb_b200_detect_result* h_results,
                                              const float** h_series, const void** d_spectrum,
                                              const srtb_b200_event** h_events, uint64_t* n_events) {
  return collect_ring(ctx, ticket, h_results, h_series, d_spectrum, true, h_events, n_events);
}

extern "C" int srtb_b200_collect_block(srtb_b200_ctx* ctx, int ticket, srtb_b200_detect_result* h_results) {
  return srtb_b200_collect_block_ex(ctx, ticket, h_results, nullptr, nullptr);
}

extern "C" const void* srtb_b200_block_spectrum(const srtb_b200_ctx* ctx, int stream) {
  if (!ctx || stream < 0 || stream >= 4) return nullptr;
  return ctx->stream_buf[stream].p;
}

// every trial of a DM sweep writes its dynamic spectrum into sweep_buf; the last one written stays there
extern "C" const void* srtb_b200_sweep_spectrum(const srtb_b200_ctx* ctx) {
  if (!ctx) return nullptr;
  return ctx->sweep_buf.p;
}

// ------------------------------------------------------------------------------------
// waterfall thumbnail (simplify_spectrum_pipe_2): see thumbnail.cuh
// ------------------------------------------------------------------------------------
extern "C" int srtb_b200_simplify_spectrum(srtb_b200_ctx* ctx, const void* d_spectrum, size_t in_width,
                                           size_t in_height, size_t out_width, size_t out_height, uint32_t argb_0,
                                           uint32_t argb_1, uint32_t argb_overflow, float* d_intensity,
                                           uint32_t* d_pixmap, float* d_average) {
  API_LOCK(ctx);
  if (!ctx || !d_spectrum || !d_intensity || !d_pixmap)
    return fail(ctx, SRTB_B200_E_INVALID, "simplify_spectrum: null argument");
  if (in_width == 0 || in_height == 0 || out_width == 0 || out_height == 0)
    return fail(ctx, SRTB_B200_E_INVALID, "simplify_spectrum: zero size");
  if (in_height > 0x7fffffffu || out_width > ((size_t)1 << 31))
    return fail(ctx, SRTB_B200_E_INVALID, "simplify_spectrum: size exceeds the launch grid");
  CK(cudaSetDevice(ctx->device));
  // G threads per output pixel, about four input cells per thread; the CTA covers 256 / G pixels of one input row
  const double ratio = (double)in_width / (double)out_width;
  int G = 1;
  while (G < 32 && 4.0 * (2 * G) <= ratio) G *= 2;
  const size_t tiles = (out_width + THUMB_THREADS / G - 1) / (THUMB_THREADS / G);
  if (tiles > 65535) return fail(ctx, SRTB_B200_E_INVALID, "simplify_spectrum: out_width too large for this in_width");
  const size_t n = out_width * out_height;
  const unsigned col_grid = (unsigned)std::min<size_t>(1024, (n + THUMB_THREADS - 1) / THUMB_THREADS);
  if (int rc = grow(ctx, ctx->thumb_rows, sizeof(float) * in_height * out_width)) return rc;
  if (int rc = grow(ctx, ctx->thumb_partial, sizeof(float) * col_grid)) return rc;

  const float2* spec = static_cast<const float2*>(d_spectrum);
  const dim3 row_grid((unsigned)in_height, (unsigned)tiles);
  const bool vec = in_width % 2 == 0 && (reinterpret_cast<uintptr_t>(d_spectrum) & 15u) == 0;
  CK(launch(ctx, false, vec ? thumb_row_kernel<true> : thumb_row_kernel<false>, row_grid, THUMB_THREADS, 0, spec,
            in_width, out_width, G, ctx->thumb_rows.p));
  CK(launch(ctx, false, thumb_col_kernel, col_grid, THUMB_THREADS, 0, ctx->thumb_rows.p, in_height, out_width, out_height,
            d_intensity, ctx->thumb_partial.p));
  CK(launch(ctx, false, thumb_norm_kernel, grid_for(ctx, n, THUMB_THREADS, 4), THUMB_THREADS, 0, d_intensity, n,
            ctx->thumb_partial.p, (int)col_grid, argb_0, argb_1, argb_overflow, d_pixmap, d_average));
  return 0;
}

// ------------------------------------------------------------------------------------
// baseband correlator (the reference's correlator.cpp): see correlator.cuh
// ------------------------------------------------------------------------------------
static int launch_cross_spectrum(srtb_b200_ctx* ctx, const float2* a, const float2* b, size_t M, float norm,
                                 float2* out) {
  const bool vec = ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) |
                     reinterpret_cast<uintptr_t>(out)) & 15u) == 0;
  CK(launch(ctx, false, vec ? cross_spectrum_kernel<true> : cross_spectrum_kernel<false>,
            grid_for(ctx, vec ? M / 2 + 1 : M, 256), 256, 0, a, b, M, norm, out));
  return 0;
}

// out[i] = |y[i]| for i < M; two bins per access when out is 8-byte aligned (y is a ctx buffer, 16-byte aligned)
static int launch_magnitude(srtb_b200_ctx* ctx, const float2* y, size_t M, float* out) {
  const bool vec = (reinterpret_cast<uintptr_t>(out) & 7u) == 0;
  CK(launch(ctx, false, vec ? magnitude_kernel<true> : magnitude_kernel<false>, grid_for(ctx, vec ? M / 2 + 1 : M, 256),
            256, 0, y, M, out));
  return 0;
}

static bool byte_ranges_overlap(const void* p, const void* q, size_t bytes) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p), b = reinterpret_cast<uintptr_t>(q);
  return a < b + bytes && b < a + bytes;
}

extern "C" int srtb_b200_cross_spectrum(srtb_b200_ctx* ctx, const void* d_a, const void* d_b, size_t count, float norm,
                                        void* d_out) {
  API_LOCK(ctx);
  if (!ctx || !d_a || !d_b || !d_out) return fail(ctx, SRTB_B200_E_INVALID, "cross_spectrum: null argument");
  if (count == 0) return fail(ctx, SRTB_B200_E_INVALID, "cross_spectrum: zero count");
  if (!aligned8(d_a) || !aligned8(d_b) || !aligned8(d_out))
    return fail(ctx, SRTB_B200_E_INVALID, "cross_spectrum: a pointer is not 8-byte aligned");
  if (count > (SIZE_MAX >> 4)) return fail(ctx, SRTB_B200_E_INVALID, "cross_spectrum: count too large");
  const size_t bytes = count * sizeof(float2);
  if ((d_out != d_a && byte_ranges_overlap(d_out, d_a, bytes)) || (d_out != d_b && byte_ranges_overlap(d_out, d_b, bytes)))
    return fail(ctx, SRTB_B200_E_INVALID, "cross_spectrum: d_out overlaps an input without being it");
  CK(cudaSetDevice(ctx->device));
  return launch_cross_spectrum(ctx, static_cast<const float2*>(d_a), static_cast<const float2*>(d_b), count, norm,
                               static_cast<float2*>(d_out));
}

extern "C" int srtb_b200_correlate(srtb_b200_ctx* ctx, const void* d_in_1, const void* d_in_2, size_t input_size,
                                   float* d_out) {
  API_LOCK(ctx);
  if (!ctx || !d_in_1 || !d_in_2 || !d_out) return fail(ctx, SRTB_B200_E_INVALID, "correlate: null argument");
  if (reinterpret_cast<uintptr_t>(d_out) & 3u)
    return fail(ctx, SRTB_B200_E_INVALID, "correlate: d_out is not 4-byte aligned");
  if (input_size < 2)
    return fail(ctx, SRTB_B200_E_INVALID, "correlate: input_size must be at least 2 bytes, got " +
                                              std::to_string(input_size));
  const size_t M = input_size / 2, N = 2 * M;  // complex_count, real_count (correlator.cpp:56-57)
  if (!is_pow2(N)) return fail(ctx, SRTB_B200_E_SIZE, "[fft] n must be a power of 2, got " + std::to_string(N));
  if (N > ((size_t)1 << 31))
    return fail(ctx, SRTB_B200_E_SIZE, "correlate: real_count " + std::to_string(N) + " above 2^31 samples not supported");
  CK(cudaSetDevice(ctx->device));
  for (auto& b : ctx->corr_buf)
    if (int rc = grow(ctx, b, (N + 2) * sizeof(float))) return rc;
  // std::pow(input_size, -1.5) in double, stored as float (correlator.cpp:59): an odd input_size counts (q13)
  const float norm = static_cast<float>(std::pow(static_cast<double>(input_size), -1.5));
  // each input is one SIMPLE stream of unsigned 8-bit samples without a window: the block path's R2C, with the unpack
  // fused into the first sweep where raw_sources_for allows it
  srtb_b200_block_config cfg{};
  cfg.baseband_input_count = N;
  cfg.baseband_input_bits = 8;
  cfg.baseband_format = SRTB_B200_FORMAT_SIMPLE;
  cfg.window = SRTB_B200_WINDOW_RECTANGLE;
  block_params p;
  p.cfg = &cfg;
  p.streams = 1;
  p.N = N;
  const void* inputs[2] = {d_in_1, d_in_2};
  for (int s = 0; s < 2; s++) {
    float* const bufs[4] = {ctx->corr_buf[s].p, nullptr, nullptr, nullptr};
    block_input in{inputs[s], N, bufs};
    if (int rc = block_input_init(ctx, p, &in)) return rc;
    if (int rc = r2c_stream(ctx, p, &in, 0, /*fork=*/false)) return rc;
  }
  // (1) cross spectrum over X1 (the Nyquist bin is dropped), (2) unnormalised backward C2C of M points, (3) |y|
  float2* x1 = reinterpret_cast<float2*>(ctx->corr_buf[0].p);
  if (int rc = launch_cross_spectrum(ctx, x1, reinterpret_cast<const float2*>(ctx->corr_buf[1].p), M, norm, x1)) return rc;
  if (int rc = fft_c2c_impl<false>(ctx, x1, M, 1)) return rc;
  return launch_magnitude(ctx, x1, M, d_out);
}

// ---- the integrating, segment-averaged correlator (see include/srtb_b200.h and correlator.cuh)

static int check_segment_size(srtb_b200_ctx* ctx, const char* who, size_t Ls) {
  if (!is_pow2(Ls) || Ls < 16 || Ls > ((size_t)1 << 30))
    return fail(ctx, SRTB_B200_E_SIZE, std::string(who) + ": segment_size must be a power of two from 16 to 2^30, got " +
                                           std::to_string(Ls));
  return 0;
}

template <int BITS>
static int launch_corr_pack(srtb_b200_ctx* ctx, const void* in_1, const void* in_2, int log_ls, size_t n_segments,
                            size_t rows, float2* out) {
  const uintptr_t group = BITS < 0 ? -BITS : BITS;  // bytes of 8 samples: unpack_src<BITS>'s load width
  const bool vec = reinterpret_cast<uintptr_t>(in_1) % group == 0 && reinterpret_cast<uintptr_t>(in_2) % group == 0;
  const size_t pairs = (2 * rows) << log_ls;
  CK(launch(ctx, false, vec ? corr_pack_kernel<BITS, true> : corr_pack_kernel<BITS, false>,
            grid_for(ctx, vec ? pairs / 8 : pairs, 256), 256, 0, in_1, in_2, log_ls, n_segments, rows, out));
  return 0;
}

extern "C" int srtb_b200_correlate_accumulate(srtb_b200_ctx* ctx, const void* d_in_1, const void* d_in_2, int bits,
                                              size_t segment_size, size_t n_segments, void* d_acc, int reset) {
  API_LOCK(ctx);
  if (!ctx || !d_in_1 || !d_in_2 || !d_acc) return fail(ctx, SRTB_B200_E_INVALID, "correlate_accumulate: null argument");
  if (bits != 1 && bits != 2 && bits != 4 && bits != 8 && bits != -8)
    return fail(ctx, SRTB_B200_E_INVALID, "correlate_accumulate: bits must be 1, 2, 4, 8 or -8, got " +
                                              std::to_string(bits));
  if (n_segments == 0) return fail(ctx, SRTB_B200_E_INVALID, "correlate_accumulate: n_segments is zero");
  if (reinterpret_cast<uintptr_t>(d_acc) & 15u)
    return fail(ctx, SRTB_B200_E_INVALID, "correlate_accumulate: d_acc is not 16-byte aligned");
  if (int rc = check_segment_size(ctx, "correlate_accumulate", segment_size)) return rc;
  if (n_segments > ((size_t)1 << 34) / segment_size)
    return fail(ctx, SRTB_B200_E_SIZE, "correlate_accumulate: n_segments * segment_size above 2^34");
  CK(cudaSetDevice(ctx->device));
  const size_t Ls = segment_size, Ms = Ls / 2, rows = (n_segments + 1) / 2;  // rows per input
  const int log_ls = ilog2(Ls);
  if (int rc = grow(ctx, ctx->corr_rows, 2 * rows * Ls * sizeof(float2))) return rc;
  const unsigned target = (unsigned)ctx->sm_count * 8;  // resident 256-thread CTAs of the whole GPU
  if (!ctx->corr_tickets) {
    CK(cudaMalloc(&ctx->corr_tickets, target * sizeof(unsigned)));
    CK(cudaMemsetAsync(ctx->corr_tickets, 0, target * sizeof(unsigned), ctx->lane.stream));
  }
  float2* z = ctx->corr_rows.p;
  int rc = 0;
  switch (bits) {
    case 1: rc = launch_corr_pack<1>(ctx, d_in_1, d_in_2, log_ls, n_segments, rows, z); break;
    case 2: rc = launch_corr_pack<2>(ctx, d_in_1, d_in_2, log_ls, n_segments, rows, z); break;
    case 4: rc = launch_corr_pack<4>(ctx, d_in_1, d_in_2, log_ls, n_segments, rows, z); break;
    case 8: rc = launch_corr_pack<8>(ctx, d_in_1, d_in_2, log_ls, n_segments, rows, z); break;
    default: rc = launch_corr_pack<-8>(ctx, d_in_1, d_in_2, log_ls, n_segments, rows, z); break;
  }
  if (rc) return rc;
  if (int rc2 = fft_c2c_impl<true>(ctx, z, Ls, 2 * rows)) return rc2;
  // split grid: bin tiles of BT bins x row groups. More than one group only when the tiles alone cannot fill the GPU;
  // then tiles < target, so the target tickets suffice.
  const int log_bt = std::min(log_ls - 1, 8);
  const size_t BT = (size_t)1 << log_bt, tiles = Ms / BT, lanes = 256 / BT;
  size_t groups = 1;
  if (tiles < target) groups = std::min((target + tiles - 1) / tiles, (rows + lanes - 1) / lanes);
  const size_t rows_per_group = (rows + groups - 1) / groups;
  groups = (rows + rows_per_group - 1) / rows_per_group;
  double2* partial = nullptr;
  if (groups > 1) {
    if (int rc2 = grow(ctx, ctx->corr_partial, groups * Ms * sizeof(double2))) return rc2;
    partial = ctx->corr_partial.p;
  }
  CK(launch(ctx, false, corr_split_accumulate_kernel, dim3((unsigned)tiles, (unsigned)groups), 256, 0, z, log_ls, log_bt,
            rows, n_segments, rows_per_group, partial, ctx->corr_tickets, static_cast<double2*>(d_acc), reset));
  return 0;
}

extern "C" int srtb_b200_correlate_finish(srtb_b200_ctx* ctx, const void* d_acc, size_t segment_size,
                                          uint64_t total_segments, float* d_out) {
  API_LOCK(ctx);
  if (!ctx || !d_acc || !d_out) return fail(ctx, SRTB_B200_E_INVALID, "correlate_finish: null argument");
  if (total_segments == 0) return fail(ctx, SRTB_B200_E_INVALID, "correlate_finish: total_segments is zero");
  if (reinterpret_cast<uintptr_t>(d_acc) & 15u)
    return fail(ctx, SRTB_B200_E_INVALID, "correlate_finish: d_acc is not 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(d_out) & 3u)
    return fail(ctx, SRTB_B200_E_INVALID, "correlate_finish: d_out is not 4-byte aligned");
  if (int rc = check_segment_size(ctx, "correlate_finish", segment_size)) return rc;
  CK(cudaSetDevice(ctx->device));
  const size_t Ms = segment_size / 2;
  if (int rc = grow(ctx, ctx->corr_rows, Ms * sizeof(float2))) return rc;
  // the reference's norm with Ls in place of input_size, rounded to float, then over the segment count in float64
  const float norm = static_cast<float>(std::pow(static_cast<double>(segment_size), -1.5));
  const double scale = static_cast<double>(norm) / static_cast<double>(total_segments);
  float2* y = ctx->corr_rows.p;
  CK(launch(ctx, false, corr_scale_kernel, grid_for(ctx, Ms, 256), 256, 0, static_cast<const double2*>(d_acc), Ms, scale,
            y));
  if (int rc = fft_c2c_impl<false>(ctx, y, Ms, 1)) return rc;
  return launch_magnitude(ctx, y, Ms, d_out);
}
