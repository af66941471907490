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
#include <set>
#include <string>
#include <vector>

#include "../../include/srtb_b200.h"
#include "fft_engine.cuh"
#include "fft_bigrow.cuh"
#include "ops_kernels.cuh"

using namespace srtb_b200;

static thread_local std::string g_last_error;

struct srtb_b200_ctx {
  // a context may be shared by the threads of a pipeline (the reference hands one sycl::queue to every pipe): every
  // C-ABI entry takes this lock, so the planning state below (tables, scratch sizes, kernel attributes) is never
  // mutated concurrently. Recursive because the block entries call the stage entries.
  std::recursive_mutex mu;
  int device = 0;
  cudaStream_t stream = nullptr;
  int sm_count = 132;
  std::string err;
  uint64_t launches = 0;
  std::set<const void*> configured;  // kernels whose smem attribute is set on this device
  std::map<const void*, int> occupancy;  // resident CTAs per SM of the persistent kernels
  // FFT
  float2* tw[13] = {nullptr};
  std::map<int, float2*> bigtw;  // log2(n_i) -> [3 << q]
  float2* bigrow_tab[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};  // [logl - 13][forward] whole-row kernel tables
  void* fft_scratch = nullptr;
  size_t fft_scratch_bytes = 0;
  // s1
  double* partial = nullptr;
  unsigned* ticket = nullptr;
  unsigned* detect_ticket = nullptr;  // last-CTA ticket of the detector's column-sum kernel
  float* mean = nullptr;
  // detect (slots = streams in flight)
  float* colsum_partial = nullptr;
  size_t colsum_partial_elems = 0;
  float* series[4] = {nullptr, nullptr, nullptr, nullptr};
  size_t series_elems = 0;
  float* acc = nullptr;
  size_t acc_elems = 0;
  detect_dev_result* d_res = nullptr;
  detect_dev_result* h_res = nullptr;  // pinned, 4 slots
  size_t slot_time_count[4] = {0, 0, 0, 0};
  // pipelined ingest ring
  cudaStream_t copy_stream = nullptr;
  void* slot_baseband[SRTB_B200_RING_SLOTS] = {nullptr};
  size_t slot_baseband_bytes[SRTB_B200_RING_SLOTS] = {0};
  cudaEvent_t slot_h2d[SRTB_B200_RING_SLOTS] = {nullptr}, slot_done[SRTB_B200_RING_SLOTS] = {nullptr};
  int slot_streams[SRTB_B200_RING_SLOTS] = {0};
  size_t slot_L[SRTB_B200_RING_SLOTS] = {0};
  bool slot_busy[SRTB_B200_RING_SLOTS] = {false};
  cudaEvent_t slot_done_alt[SRTB_B200_RING_SLOTS] = {nullptr};  // second lane's completion of the slot's block
  bool slot_alt_used[SRTB_B200_RING_SLOTS] = {false};
  int slot_ticket[SRTB_B200_RING_SLOTS] = {0};
  // per-slot outputs: ctx-owned working buffers / pinned series unless the caller supplied its own (submit_block_ex)
  float* slot_stream_buf[SRTB_B200_RING_SLOTS][4] = {};
  size_t slot_stream_elems[SRTB_B200_RING_SLOTS] = {0};
  float* slot_h_series[SRTB_B200_RING_SLOTS] = {nullptr};
  size_t slot_h_series_elems[SRTB_B200_RING_SLOTS] = {0};
  float* slot_out_spectrum[SRTB_B200_RING_SLOTS][4] = {};
  float* slot_out_series[SRTB_B200_RING_SLOTS] = {nullptr};
  uint64_t submit_count = 0;
  // DM sweep working copy of the spectrum, per-trial result headers
  void* sweep_buf = nullptr;
  size_t sweep_buf_bytes = 0;
  void* sweep_res = nullptr;
  size_t sweep_res_bytes = 0;
  // long waterfall rows: per-tile SK statistics of the last sweep, per-row zap flags
  void* long_stats = nullptr;
  size_t long_stats_bytes = 0;
  void* long_zap = nullptr;
  size_t long_zap_bytes = 0;
  // optional per-stage timing (srtb_b200_stage_stats)
  bool stats_on = false;
  cudaEvent_t stat_ev[SRTB_B200_STAGE_COUNT][2] = {};
  double stat_bytes[SRTB_B200_STAGE_COUNT] = {};
  bool stat_have[SRTB_B200_STAGE_COUNT] = {};
  // ring path: pinned host destination [streams][MAX_BOXCARS][L] of the current block's positive series (else null)
  float* host_series_dst = nullptr;
  bool pdl_auto = false;    // programmatic dependent launch for the current block (short kernels only)
  bool res_zeroed = false;  // block path: the per-stream result headers were zeroed before the first kernel
  // process_block
  void* d_baseband = nullptr;
  size_t d_baseband_bytes = 0;
  float* stream_buf[4] = {nullptr, nullptr, nullptr, nullptr};
  size_t stream_buf_elems = 0;
  // K12 phase table of the current (block geometry, DM): see chirp_phase_table_kernel
  float* chirp_tab = nullptr;
  size_t chirp_tab_bytes = 0;
  double chirp_tab_key[6] = {0, 0, 0, 0, 0, 0};  // n, f_min, df, inv_fc, f_c, ddm
  // second lane: the data streams of one block are independent until their result headers are read back, so the
  // odd-numbered ones run on a second CUDA stream of this context with their own scratch (one lane's kernel tails and
  // small detector kernels overlap the other lane's FFT sweeps). lane_swap() exchanges every member a stream's chain
  // writes through with the copy kept here, so the launch code itself is lane-agnostic.
  struct lane_state {
    cudaStream_t stream = nullptr;
    void* fft_scratch = nullptr;
    size_t fft_scratch_bytes = 0;
    double* partial = nullptr;
    unsigned* ticket = nullptr;
    unsigned* detect_ticket = nullptr;
    float* mean = nullptr;
    float* colsum_partial = nullptr;
    size_t colsum_partial_elems = 0;
    float* acc = nullptr;
    size_t acc_elems = 0;
    void* long_stats = nullptr;
    size_t long_stats_bytes = 0;
    void* long_zap = nullptr;
    size_t long_zap_bytes = 0;
  } alt;
  bool alt_ready = false, on_alt = false;
  int lanes = 1;  // SRTB_B200_LANES (default 2): CUDA streams per context the data streams of a block are spread over
  cudaEvent_t lane_fork = nullptr, lane_join = nullptr;
};

static void lane_swap(srtb_b200_ctx* ctx) {
  auto& a = ctx->alt;
  std::swap(ctx->stream, a.stream);
  std::swap(ctx->fft_scratch, a.fft_scratch);
  std::swap(ctx->fft_scratch_bytes, a.fft_scratch_bytes);
  std::swap(ctx->partial, a.partial);
  std::swap(ctx->ticket, a.ticket);
  std::swap(ctx->detect_ticket, a.detect_ticket);
  std::swap(ctx->mean, a.mean);
  std::swap(ctx->colsum_partial, a.colsum_partial);
  std::swap(ctx->colsum_partial_elems, a.colsum_partial_elems);
  std::swap(ctx->acc, a.acc);
  std::swap(ctx->acc_elems, a.acc_elems);
  std::swap(ctx->long_stats, a.long_stats);
  std::swap(ctx->long_stats_bytes, a.long_stats_bytes);
  std::swap(ctx->long_zap, a.long_zap);
  std::swap(ctx->long_zap_bytes, a.long_zap_bytes);
  ctx->on_alt = !ctx->on_alt;
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
  CK(cudaStreamSynchronize(ctx->stream));
  if (ctx->alt_ready) CK(cudaStreamSynchronize(ctx->alt.stream));
  return 0;
}

static int ensure(srtb_b200_ctx* ctx, void** p, size_t* have, size_t want_bytes) {
  if (*have >= want_bytes && *p) return 0;
  if (*p) {
    if (int rc = sync_lanes(ctx)) return rc;
    CK(cudaFree(*p));
    *p = nullptr;
    *have = 0;
  }
  cudaError_t e = cudaMalloc(p, want_bytes);
  if (e != cudaSuccess)
    return fail(ctx, SRTB_B200_E_NOMEM, std::string("cudaMalloc(") + std::to_string(want_bytes) +
                                            "): " + cudaGetErrorString(e));
  *have = want_bytes;
  return 0;
}

static inline bool is_pow2(size_t n) { return n && !(n & (n - 1)); }
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
    cudaEventRecord(ctx->stat_ev[stage][0], ctx->stream);
  }
  ~stage_scope() {
    if (ctx) cudaEventRecord(ctx->stat_ev[stage][1], ctx->stream);
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
  ctx->stream = static_cast<cudaStream_t>(cuda_stream);
  e = cudaSetDevice(device);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device);
  if (e == cudaSuccess) e = cudaMalloc(&ctx->partial, sizeof(double) * 4096);
  if (e == cudaSuccess) e = cudaMalloc(&ctx->ticket, sizeof(unsigned));
  if (e == cudaSuccess) e = cudaMemset(ctx->ticket, 0, sizeof(unsigned));
  if (e == cudaSuccess) e = cudaMalloc(&ctx->detect_ticket, sizeof(unsigned));
  if (e == cudaSuccess) e = cudaMemset(ctx->detect_ticket, 0, sizeof(unsigned));
  if (e == cudaSuccess) e = cudaMalloc(&ctx->mean, sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&ctx->d_res, sizeof(detect_dev_result) * 4);
  if (e == cudaSuccess) e = cudaMemset(ctx->d_res, 0, sizeof(detect_dev_result) * 4);
  if (e == cudaSuccess) e = cudaMallocHost(&ctx->h_res, sizeof(detect_dev_result) * 4 * (1 + SRTB_B200_RING_SLOTS));
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
  cudaStreamSynchronize(ctx->stream);
  if (ctx->alt_ready) {
    cudaStreamSynchronize(ctx->alt.stream);
    cudaFree(ctx->alt.fft_scratch);
    cudaFree(ctx->alt.partial);
    cudaFree(ctx->alt.ticket);
    cudaFree(ctx->alt.detect_ticket);
    cudaFree(ctx->alt.mean);
    cudaFree(ctx->alt.colsum_partial);
    cudaFree(ctx->alt.acc);
    cudaFree(ctx->alt.long_stats);
    cudaFree(ctx->alt.long_zap);
    cudaStreamDestroy(ctx->alt.stream);
  }
  if (ctx->lane_fork) cudaEventDestroy(ctx->lane_fork);
  if (ctx->lane_join) cudaEventDestroy(ctx->lane_join);
  for (auto& p : ctx->tw)
    if (p) cudaFree(p);
  for (auto& kv : ctx->bigtw) cudaFree(kv.second);
  for (auto& a : ctx->bigrow_tab)
    for (auto& p : a) cudaFree(p);
  cudaFree(ctx->fft_scratch);
  cudaFree(ctx->partial);
  cudaFree(ctx->ticket);
  cudaFree(ctx->detect_ticket);
  cudaFree(ctx->mean);
  cudaFree(ctx->colsum_partial);
  for (auto& p : ctx->series) cudaFree(p);
  cudaFree(ctx->acc);
  cudaFree(ctx->d_res);
  cudaFreeHost(ctx->h_res);
  cudaFree(ctx->d_baseband);
  cudaFree(ctx->sweep_buf);
  cudaFree(ctx->sweep_res);
  cudaFree(ctx->long_stats);
  cudaFree(ctx->long_zap);
  cudaFree(ctx->chirp_tab);
  for (int i = 0; i < SRTB_B200_RING_SLOTS; i++) {
    cudaFree(ctx->slot_baseband[i]);
    for (auto& p : ctx->slot_stream_buf[i]) cudaFree(p);
    if (ctx->slot_h_series[i]) cudaFreeHost(ctx->slot_h_series[i]);
    if (ctx->slot_h2d[i]) cudaEventDestroy(ctx->slot_h2d[i]);
    if (ctx->slot_done[i]) cudaEventDestroy(ctx->slot_done[i]);
    if (ctx->slot_done_alt[i]) cudaEventDestroy(ctx->slot_done_alt[i]);
  }
  if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
  for (auto& p : ctx->stream_buf) cudaFree(p);
  for (auto& ev : ctx->stat_ev)
    for (auto& e2 : ev)
      if (e2) cudaEventDestroy(e2);
  delete ctx;
  return 0;
}

int srtb_b200_ctx_set_stream(srtb_b200_ctx* ctx, void* cuda_stream) {
  API_LOCK(ctx);
  if (!ctx) return fail(nullptr, SRTB_B200_E_INVALID, "set_stream: ctx is null");
  ctx->stream = static_cast<cudaStream_t>(cuda_stream);
  return 0;
}

int srtb_b200_synchronize(srtb_b200_ctx* ctx) {
  if (!ctx) return fail(nullptr, SRTB_B200_E_INVALID, "synchronize: ctx is null");
  cudaStream_t s0, s1 = nullptr;
  {
    API_LOCK(ctx);  // the wait itself runs unlocked: other threads keep enqueueing meanwhile
    s0 = ctx->on_alt ? ctx->alt.stream : ctx->stream;
    if (ctx->alt_ready) s1 = ctx->on_alt ? ctx->stream : ctx->alt.stream;
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
    unpack_simple_scalar_kernel<BITS><<<grid_for(ctx, n, 256), 256, 0, ctx->stream>>>(d_in, out, n, window);
  } else if (window == 0) {
    unpack_simple_kernel<BITS, false><<<grid_for(ctx, n / 16 + 1, 256), 256, 0, ctx->stream>>>(d_in, out, n, window);
  } else {
    unpack_simple_kernel<BITS, true><<<grid_for(ctx, n / 16 + 1, 256), 256, 0, ctx->stream>>>(d_in, out, n, window);
  }
  ctx->launches++;
  CK(cudaGetLastError());
  return 0;
}

template <int BITS>
static int launch_unpack_il2(srtb_b200_ctx* ctx, const void* d_in, float* o1, float* o2, size_t n, int window) {
  unpack_interleaved2_kernel<BITS><<<grid_for(ctx, n / 4 + 1, 256), 256, 0, ctx->stream>>>(d_in, o1, o2, n, window);
  ctx->launches++;
  CK(cudaGetLastError());
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
      unpack_snap1_kernel<<<grid_for(ctx, out_count / 4 + 1, 256), 256, 0, ctx->stream>>>(d_in, d_out[0], d_out[1], out_count, window);
      break;
    case SRTB_B200_FORMAT_GZNUPSR_A1_2:
      unpack_gznupsr_kernel<2><<<grid_for(ctx, out_count / 4 + 1, 256), 256, 0, ctx->stream>>>(
          d_in, d_out[0], d_out[1], nullptr, nullptr, out_count, window);
      break;
    case SRTB_B200_FORMAT_GZNUPSR_A1_4:
      unpack_gznupsr_kernel<4><<<grid_for(ctx, out_count / 4 + 1, 256), 256, 0, ctx->stream>>>(
          d_in, d_out[0], d_out[1], d_out[2], d_out[3], out_count, window);
      break;
  }
  ctx->launches++;
  CK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------
// FFT planning + launches
// ------------------------------------------------------------------------------------
static int get_stage_twiddles(srtb_b200_ctx* ctx, int logl, const float2** out) {
  if (!ctx->tw[logl]) {
    const size_t L = (size_t)1 << logl;
    std::vector<float2> h(L);
    for (size_t j = 0; j < L; j++) {
      const double a = -2.0 * M_PI * (double)j / (double)L;
      h[j] = make_float2((float)std::cos(a), (float)std::sin(a));
    }
    CK(cudaMalloc(&ctx->tw[logl], L * sizeof(float2)));
    CK(cudaMemcpyAsync(ctx->tw[logl], h.data(), L * sizeof(float2), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  *out = ctx->tw[logl];
  return 0;
}

static int get_big_twiddles(srtb_b200_ctx* ctx, int logn, big_twiddle* out) {
  const int q = (logn + 2) / 3;
  auto it = ctx->bigtw.find(logn);
  if (it == ctx->bigtw.end()) {
    const size_t n = (size_t)1 << logn, m = (size_t)1 << q;
    std::vector<float2> h(3 * m);
    for (int level = 0; level < 3; level++)
      for (size_t j = 0; j < m; j++) {
        const size_t idx = (j << (level * q)) & (n - 1);
        const double a = -2.0 * M_PI * (double)idx / (double)n;
        h[level * m + j] = make_float2((float)std::cos(a), (float)std::sin(a));
      }
    float2* d = nullptr;
    CK(cudaMalloc(&d, h.size() * sizeof(float2)));
    CK(cudaMemcpyAsync(d, h.data(), h.size() * sizeof(float2), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    it = ctx->bigtw.emplace(logn, d).first;
  }
  out->tab = it->second;
  out->q = q;
  return 0;
}

template <int LOGL, int T, int MODE, bool FWD, class IO>
static int launch_pass(srtb_b200_ctx* ctx, const IO& io, unsigned grid, size_t extra_smem) {
  auto kern = fft_pass_kernel<LOGL, T, MODE, FWD, IO>;
  const size_t smem = (size_t)tile_layout<LOGL, T, MODE>::ELEMS * sizeof(float2) + extra_smem;
  const void* key = reinterpret_cast<const void*>(kern);
  if (smem > 48 * 1024 && !ctx->configured.count(key)) {
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(200 * 1024)));
    ctx->configured.insert(key);
  }
  const float2* tw = nullptr;
  if (int rc = get_stage_twiddles(ctx, LOGL, &tw)) return rc;
  kern<<<grid, pass_threads<LOGL, T>::value, smem, ctx->stream>>>(io, tw);
  ctx->launches++;
  CK(cudaGetLastError());
  return 0;
}

// rows per CTA in ROW mode: 256 threads up to L = 2048, 512 threads for L = 4096
template <int LOGL>
struct row_t {
  static constexpr int value = (LOGL >= 11) ? 1 : (1 << (11 - LOGL));
};
#ifndef SRTB_COL_T
#define SRTB_COL_T 16
#endif
template <int LOGL>
struct col_t {
  static constexpr int value = (LOGL <= 8) ? SRTB_COL_T : ((SRTB_COL_T < 8) ? SRTB_COL_T : 8);
};

// sixteen-points-per-thread row kernels (L = 256, 1024, 2048, 4096); SRTB_B200_ROW16=0 selects the
// eight-point kernels (A/B measurements)
static bool use_row16() {
  static const bool on = [] {
    const char* e = std::getenv("SRTB_B200_ROW16");
    return !(e && e[0] == '0');
  }();
  return on;
}
template <int LOGL>
struct has_row16 {
  static constexpr bool value = (LOGL >= 8 && LOGL <= 12);
};

template <int LOGL, bool FWD>
static int launch_row(srtb_b200_ctx* ctx, const float2* in, float2* out, size_t nrows) {
  constexpr int T = row_t<LOGL>::value;
  if constexpr (has_row16<LOGL>::value) {
    if ((reinterpret_cast<uintptr_t>(in) & 15u) == 0 && use_row16()) {
      constexpr int T16 = row16_t<LOGL>::value, threads = ((1 << LOGL) / 16) * T16;
      auto kern = fft_row16_tma_kernel<LOGL, T16, FWD>;
      constexpr size_t smem = row16_smem<LOGL, T16>::bytes;
      const size_t ntiles = (nrows + T16 - 1) / T16;
      unsigned grid = 1;
      if (int rc = persistent_grid(ctx, kern, threads, smem, smem, ntiles, &grid)) return rc;
      const float2* tw = nullptr;
      if (int rc = get_stage_twiddles(ctx, LOGL, &tw)) return rc;
      CK(launch_pdl(ctx, kern, dim3(grid), dim3(threads), smem, in, out, nrows, tw, row_sk_params{}, row_chirp_params{}));
      ctx->launches++;
      CK(cudaGetLastError());
      return 0;
    }
  }
  if ((reinterpret_cast<uintptr_t>(in) & 15u) == 0) {
    // persistent TMA-fed kernel (cp.async.bulk needs 16-byte aligned rows)
    auto kern = fft_row_tma_kernel<LOGL, T, FWD>;
    constexpr size_t smem = row_tma_smem<LOGL, T>::bytes;
    const void* key = reinterpret_cast<const void*>(kern);
    if (!ctx->configured.count(key)) {
      CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      int per_sm = 1;
      CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, pass_threads<LOGL, T>::value, smem));
      ctx->occupancy[key] = std::max(1, per_sm);
      ctx->configured.insert(key);
    }
    const float2* tw = nullptr;
    if (int rc = get_stage_twiddles(ctx, LOGL, &tw)) return rc;
    const size_t ntiles = (nrows + T - 1) / T;
    const unsigned grid = (unsigned)std::min<size_t>(ntiles, (size_t)ctx->sm_count * ctx->occupancy[key]);
    kern<<<grid, pass_threads<LOGL, T>::value, smem, ctx->stream>>>(in, out, nrows, tw, row_sk_params{});
    ctx->launches++;
    CK(cudaGetLastError());
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
                            CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_INT64) {
  encode_tiled_fn enc = get_encode_tiled();
  if (!enc) return false;
  static_assert(sizeof(CUtensorMap) <= sizeof(tensor_map_blob), "tensor map size");
  cuuint32_t estr[3] = {1, 1, 1};
  CUtensorMap m;
  const CUresult r = enc(&m, dtype, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes,
                         box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return false;
  std::memcpy(out->bytes, &m, sizeof(m));
  return true;
}

// Programmatic dependent launch along the block path: each kernel's set-up (tables into shared memory, barriers) overlaps
// its predecessor's tail; every such kernel calls pdl_wait() before touching anything a predecessor produces. It pays
// where kernels are short (2^24-sample blocks) and can cost where they are long, since the
// early-resident CTAs of the next kernel only take shared memory from the running one. Hence: on for blocks up to 2^25
// samples, off above; SRTB_B200_PDL=0 / 1 forces it.
static bool use_pdl(const srtb_b200_ctx* ctx) {
  static const int forced = [] {
    const char* e = std::getenv("SRTB_B200_PDL");
    return e ? (e[0] == '0' ? 0 : 1) : -1;
  }();
  return forced >= 0 ? forced == 1 : ctx->pdl_auto;
}
template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl(srtb_b200_ctx* ctx, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = ctx->stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = use_pdl(ctx) ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}

template <class K>
static int persistent_grid(srtb_b200_ctx* ctx, K kern, int threads, size_t smem, size_t smem_max, size_t ntiles,
                           unsigned* grid) {
  const void* key = reinterpret_cast<const void*>(kern);
  if (!ctx->configured.count(key)) {
    // the attribute is set once per kernel: use the largest size any later launch can ask for
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max));
    int per_sm = 1;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem));
    ctx->occupancy[key] = std::max(1, per_sm);
    ctx->configured.insert(key);
  }
  *grid = (unsigned)std::min<size_t>(ntiles, (size_t)ctx->sm_count * ctx->occupancy[key]);
  return 0;
}

// three-sweep factorisation of 2^q: the first sweep takes ceil(q/3); of the rest the longer half goes to the
// LAST sweep (2^23 = 2^8 * 2^7 * 2^8) so that the transposing pass runs as 16 x 16; SRTB_B200_PLAN_878=0
// gives the longer half to the middle sweep instead (8, 8, 7)
static bool plan_last_long() {
  static const bool on = [] {
    const char* e = std::getenv("SRTB_B200_PLAN_878");
    return !(e && e[0] == '0');
  }();
  return on;
}
// SRTB_B200_PLAN_FIRST_SHORT=1: give the FIRST sweep the short factor (2^25 = 2^8 * 2^9 * 2^8 instead of 2^9 * 2^8 * 2^8):
// the raw-byte first sweep then runs 256-point columns of 16 neighbours (64-byte raw segments for two streams)
static bool plan_first_short() {
  static const bool on = [] {
    const char* e = std::getenv("SRTB_B200_PLAN_FIRST_SHORT");
    return e && e[0] == '1';
  }();
  return on;
}
static void plan3(int q, int* l1, int* l2, int* l3) {
  *l1 = plan_first_short() ? q / 3 : (q + 2) / 3;
  const int big = (q - *l1 + 1) / 2, small = q - *l1 - big;
  // the fused R2C last sweep exists up to L = 256: keep the last factor <= 8 when one of the two is
  const bool last_big = plan_last_long() && big <= 8;
  *l2 = last_big ? small : big;
  *l3 = last_big ? big : small;
}

// 2^27 points and above: four sweeps of L <= 256 (all on the sixteen-point kernels, each near the HBM roofline)
// beat three sweeps with 512/1024-point columns; the last factor is 7 or 8 so the fused R2C last sweep applies.
// 27 = 7+7+6+7, 28 = 7+7+7+7, 29 = 7+7+7+8, 30 = 8+7+7+8. SRTB_B200_FOUR_SWEEPS=0 keeps three sweeps.
static void plan4(int q, int* l) {
  l[3] = (q >= 29) ? 8 : 7;
  int r = q - l[3];
  l[0] = (r + 2) / 3;
  l[1] = (r - l[0] + 1) / 2;
  l[2] = r - l[0] - l[1];
}
static bool use_col16();
static encode_tiled_fn get_encode_tiled();
static bool four_sweeps(int q, const void* ptr) {
  static const bool on = [] {
    const char* e = std::getenv("SRTB_B200_FOUR_SWEEPS");
    return !(e && e[0] == '0');
  }();
  return on && q >= 27 && q <= 30 && use_col16() && get_encode_tiled() != nullptr &&
         (reinterpret_cast<uintptr_t>(ptr) & 15u) == 0;
}

// sixteen-points-per-thread column kernels (radix 16 x 16 / 16 x 8) for L = 256 / 128; SRTB_B200_COL16=0
// selects the eight-point kernels instead (A/B measurements)
static bool use_col16() {
  static const bool on = [] {
    const char* e = std::getenv("SRTB_B200_COL16");
    return !(e && e[0] == '0');
  }();
  return on;
}

// wide tiles (32 neighbouring columns = 256-byte segments) for the 128-point column sweep of very long transforms,
// whose row stride is megabytes: fewer DRAM page openings / TLB entries per byte. SRTB_B200_WIDE_COL=0 disables.
static bool wide_col(size_t A, size_t L, size_t B) {
  static const bool on = [] {
    const char* e = std::getenv("SRTB_B200_WIDE_COL");
    return !(e && e[0] == '0');
  }();
  return on && B >= ((size_t)1 << 14) && A * L * B >= ((size_t)1 << 26);
}

template <int LOGL, bool FWD, int TT = col_t<LOGL>::value>
static int launch_col_tma(srtb_b200_ctx* ctx, const float2* in, float2* out, size_t A, size_t B, bool* done,
                          const row_chirp_params* chirp = nullptr) {
  constexpr int T = TT, L = 1 << LOGL;
  if constexpr (LOGL == 7 && TT == col_t<LOGL>::value) {
    if (use_col16() && wide_col(A, L, B) && !chirp) return launch_col_tma<LOGL, FWD, 32>(ctx, in, out, A, B, done);
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
    if (use_col16()) {
      auto kern16 = fft_col16_tma_kernel<LOGL, T, FWD>;
      constexpr int threads = col16_threads<LOGL, T>::value;
      const size_t smem16 = col16_smem<LOGL, T, false>::bytes(btw.q);
      if (int rc = persistent_grid(ctx, kern16, threads, smem16, col16_smem<LOGL, T, false>::bytes(10), ntiles, &grid)) return rc;
      if constexpr (!FWD) {
        if (chirp) {  // s1 + chirp applied as the tile is read (long waterfall rows)
          auto kernc = fft_col16_tma_kernel<LOGL, T, FWD, 0, true>;
          if (int rc = persistent_grid(ctx, kernc, threads, smem, tile_tma_smem<LOGL, T>::bytes(10), ntiles, &grid)) return rc;
          CK(launch_pdl(ctx, kernc, dim3(grid), dim3(threads), smem, tm, out, B, (uint32_t)(B / T), (uint32_t)ntiles, btw, tw,
                        raw_params{}, *chirp));
          ctx->launches++;
          CK(cudaGetLastError());
          *done = true;
          return 0;
        }
      }
      CK(launch_pdl(ctx, kern16, dim3(grid), dim3(threads), smem16, tm, out, B, (uint32_t)(B / T), (uint32_t)ntiles, btw, tw,
                    raw_params{}, row_chirp_params{}));
      ctx->launches++;
      CK(cudaGetLastError());
      *done = true;
      return 0;
    }
  }
  if (chirp) return 0;  // the chirp-on-load sweep exists for the sixteen-point kernel only
  auto kern = fft_col_tma_kernel<LOGL, T, FWD>;
  if (int rc = persistent_grid(ctx, kern, pass_threads<LOGL, T>::value, smem, tile_tma_smem<LOGL, T>::bytes(10), ntiles, &grid)) return rc;
  kern<<<grid, pass_threads<LOGL, T>::value, smem, ctx->stream>>>(tm, out, B, (uint32_t)(B / T), (uint32_t)ntiles, btw, tw, raw_params{});
  ctx->launches++;
  CK(cudaGetLastError());
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

template <int LOGL, int RAW, int TT = col_t<LOGL>::value>
static int launch_col_tma_raw(srtb_b200_ctx* ctx, const raw_source& src, float2* out, size_t B, bool* done) {
  constexpr int T = TT, L = 1 << LOGL;
  if constexpr (LOGL == 7 && TT == col_t<LOGL>::value) {
    if (use_col16() && wide_col(1, L, B)) return launch_col_tma_raw<LOGL, RAW, 32>(ctx, src, out, B, done);
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
  if constexpr (LOGL >= 7 && LOGL <= 9) {
    if (use_col16()) {
      auto kern16 = fft_col16_tma_kernel<LOGL, T, true, RAW>;
      constexpr int threads = col16_threads<LOGL, T>::value;
      constexpr size_t smem16 = raw16_smem<LOGL, T>::bytes;  // inter-sweep tables stay in global memory here
      if (int rc = persistent_grid(ctx, kern16, threads, smem16, smem16, ntiles, &grid)) return rc;
      CK(launch_pdl(ctx, kern16, dim3(grid), dim3(threads), smem16, tm, out, B, (uint32_t)(B / T), (uint32_t)ntiles, btw, tw, rp,
                    row_chirp_params{}));
      ctx->launches++;
      CK(cudaGetLastError());
      *done = true;
      return 0;
    }
  }
  if constexpr (RAW == 3) {
    return 0;  // packed samples: sixteen-point kernel only
  } else {
    if (src.delta) return 0;
    auto kern = fft_col_tma_kernel<LOGL, T, true, RAW>;
    if (int rc = persistent_grid(ctx, kern, pass_threads<LOGL, T>::value, smem, tile_tma_smem<LOGL, T>::bytes(10), ntiles, &grid)) return rc;
    kern<<<grid, pass_threads<LOGL, T>::value, smem, ctx->stream>>>(tm, out, B, (uint32_t)(B / T), (uint32_t)ntiles, btw, tw, rp);
    ctx->launches++;
    CK(cudaGetLastError());
    *done = true;
    return 0;
  }
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
    case 10: return src.is_signed ? launch_col_tma_raw<10, 1>(ctx, src, out, B, done) : launch_col_tma_raw<10, 2>(ctx, src, out, B, done);
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
  if constexpr ((LOGL == 7 || LOGL == 8) && T == 16) {
    if (use_col16()) {
      auto kern16 = fft_trans16_tma_kernel<LOGL, T, FWD>;
      constexpr int threads = T * (L / 16);
      const size_t smem16 = tile_tma_smem<LOGL, T>::bytes(0);
      const size_t k1tiles16 = L1 / T, ntiles16 = batch * S * k1tiles16;
      unsigned grid16 = 1;
      if (int rc = persistent_grid(ctx, kern16, threads, smem16, smem16, ntiles16, &grid16)) return rc;
      kern16<<<grid16, threads, smem16, ctx->stream>>>(tm, out, (uint32_t)A, (uint32_t)S, (uint32_t)L1,
                                                     (uint32_t)k1tiles16, (uint32_t)ntiles16, tw, (uint32_t)rest_inner,
                                                     tile_stats);
      ctx->launches++;
      CK(cudaGetLastError());
      *done = true;
      return 0;
    }
  }
  if (rest_inner > 1) return 0;  // only the sixteen-point kernel knows the four-sweep row order
  auto kern = fft_trans_tma_kernel<LOGL, T, FWD>;
  const size_t smem = tile_tma_smem<LOGL, T>::bytes(0);
  const size_t k1tiles = L1 / T, ntiles = batch * S * k1tiles;
  unsigned grid = 1;
  if (int rc = persistent_grid(ctx, kern, pass_threads<LOGL, T>::value, smem, smem, ntiles, &grid)) return rc;
  kern<<<grid, pass_threads<LOGL, T>::value, smem, ctx->stream>>>(tm, out, (uint32_t)A, (uint32_t)S, (uint32_t)L1,
                                                                  (uint32_t)k1tiles, (uint32_t)ntiles, tw, tile_stats);
  ctx->launches++;
  CK(cudaGetLastError());
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
// SRTB_B200_BIGROW=0 keeps the two-sweep column + transposing plan for these lengths (A/B measurements).
static bool use_bigrow() {
  static const bool on = [] {
    const char* e = std::getenv("SRTB_B200_BIGROW");
    return !(e && e[0] == '0');
  }();
  return on;
}

template <int LOGL>
static int get_bigrow_tables(srtb_b200_ctx* ctx, bool fwd, const float2** out) {
  using C = bigrow<LOGL>;
  float2*& d = ctx->bigrow_tab[LOGL - 13][fwd ? 1 : 0];
  if (!d) {
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
    CK(cudaMalloc(&d, h.size() * sizeof(float2)));
    CK(cudaMemcpyAsync(d, h.data(), h.size() * sizeof(float2), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  *out = d;
  return 0;
}

// sk != nullptr: SK + column sums in the epilogue (sk->partial is filled in here); chirp != nullptr: s1 + chirp on load
template <int LOGL, bool FWD>
static int launch_bigrow(srtb_b200_ctx* ctx, const float2* in, float2* out, size_t nrows, row_sk_params* sk,
                         const row_chirp_params* chirp, size_t* chunks_out) {
  using C = bigrow<LOGL>;
  if (nrows >= ((size_t)1 << 31)) return fail(ctx, SRTB_B200_E_SIZE, "fft: too many rows");
  const float2* tabs = nullptr;
  if (int rc = get_bigrow_tables<LOGL>(ctx, FWD, &tabs)) return rc;
  unsigned grid = 1;
  auto go = [&](auto kern, bool with_sk) -> int {
    const size_t smem = C::bytes;
    if (int rc = persistent_grid(ctx, kern, C::NT, smem, smem, nrows, &grid)) return rc;
    row_sk_params p{};
    if (with_sk) {
      size_t have = ctx->colsum_partial_elems * sizeof(float);
      if (int rc = ensure(ctx, reinterpret_cast<void**>(&ctx->colsum_partial), &have, (size_t)grid * sk->ts_count * sizeof(float)))
        return rc;
      ctx->colsum_partial_elems = have / sizeof(float);
      sk->partial = ctx->colsum_partial;
      p = *sk;
    }
    CK(launch_pdl(ctx, kern, dim3(grid), dim3(C::NT), smem, in, out, (unsigned)nrows, tabs, p, chirp ? *chirp : row_chirp_params{}));
    ctx->launches++;
    CK(cudaGetLastError());
    if (chunks_out) *chunks_out = grid;
    return 0;
  };
  if constexpr (!FWD) {
    if (sk && chirp && chirp->newton == 5) return go(fft_bigrow_kernel<LOGL, false, true, 5>, true);
    if (sk && chirp && chirp->newton == 1) return go(fft_bigrow_kernel<LOGL, false, true, 1>, true);
    if (sk && chirp && chirp->newton == 3) return go(fft_bigrow_kernel<LOGL, false, true, 3>, true);
    if (sk && chirp && chirp->newton == 4) return go(fft_bigrow_kernel<LOGL, false, true, 4>, true);
    if (sk && chirp) return go(fft_bigrow_kernel<LOGL, false, true, 2>, true);
    if (sk) return go(fft_bigrow_kernel<LOGL, false, true, 0>, true);
  }
  if (sk || chirp) return fail(ctx, SRTB_B200_E_UNSUPPORTED, "fft: fused epilogue exists for the backward transform only");
  return go(fft_bigrow_kernel<LOGL, FWD, false, 0>, false);
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
    tiny_fft_kernel<FWD><<<(unsigned)((batch + 255) / 256), 256, 0, ctx->stream>>>(x, q, batch);
    ctx->launches++;
    CK(cudaGetLastError());
    return 0;
  }
  if (q <= 12) return dispatch_row<FWD>(ctx, q, x, x, batch);
  if ((q == 13 || q == 14) && use_bigrow() && (reinterpret_cast<uintptr_t>(x) & 15u) == 0) {
    // one sweep: the whole row in shared memory (in place: a CTA reads its row completely before it stores it)
    return q == 13 ? launch_bigrow<13, FWD>(ctx, x, x, batch, nullptr, nullptr, nullptr)
                   : launch_bigrow<14, FWD>(ctx, x, x, batch, nullptr, nullptr, nullptr);
  }
  if (q > 30) return fail(ctx, SRTB_B200_E_SIZE, "fft: length above 2^30 not supported");
  if (batch * n > ((size_t)1 << 32) * 4)
    return fail(ctx, SRTB_B200_E_SIZE, "fft: batch * length too large");
  if (int rc = ensure(ctx, &ctx->fft_scratch, &ctx->fft_scratch_bytes, batch * n * sizeof(float2))) return rc;
  float2* s = static_cast<float2*>(ctx->fft_scratch);
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
  if (length == 0 || batch == 0) return fail(ctx, SRTB_B200_E_INVALID, "fft_c2c: zero size");
  if (!is_pow2(length))
    return fail(ctx, SRTB_B200_E_SIZE, "[fft] n must be a power of 2, got " + std::to_string(length));
  if (direction != 1 && direction != -1) return fail(ctx, SRTB_B200_E_INVALID, "fft_c2c: direction must be +1 / -1");
  CK(cudaSetDevice(ctx->device));
  if (direction == 1) return fft_c2c_impl<true>(ctx, static_cast<float2*>(d_x), length, batch);
  return fft_c2c_impl<false>(ctx, static_cast<float2*>(d_x), length, batch);
}

extern "C" int srtb_b200_watfft_c2c_backward(srtb_b200_ctx* ctx, void* d_x, size_t length, size_t batch) {
  API_LOCK(ctx);
  if (!ctx) return fail(nullptr, SRTB_B200_E_INVALID, "watfft: ctx is null");
  stage_scope stats_(ctx, SRTB_B200_STAGE_WATFFT, 16.0 * (double)length * (double)batch);
  return srtb_b200_fft_c2c(ctx, d_x, length, batch, -1);
}

static int fft_r2c_with_power_mean(srtb_b200_ctx* ctx, float* d_inout, size_t n_real, const raw_source* raw = nullptr,
                                   bool* raw_used = nullptr);

extern "C" int srtb_b200_fft_r2c_inplace(srtb_b200_ctx* ctx, float* d_inout, size_t n_real) {
  API_LOCK(ctx);
  if (!ctx || !d_inout) return fail(ctx, SRTB_B200_E_INVALID, "fft_r2c: null argument");
  if (n_real < 2 || !is_pow2(n_real))
    return fail(ctx, SRTB_B200_E_SIZE, "[fft] n must be a power of 2, got " + std::to_string(n_real));
  CK(cudaSetDevice(ctx->device));
  const size_t M = n_real / 2;
  stage_scope stats_(ctx, SRTB_B200_STAGE_FFT_R2C, 8.0 * (double)n_real);
  if (M >= ((size_t)1 << 13) && (reinterpret_cast<uintptr_t>(d_inout) & 15u) == 0)
    return fft_r2c_with_power_mean(ctx, d_inout, n_real);  // multi-sweep sizes: split fused into the last sweep
  float2* H = reinterpret_cast<float2*>(d_inout);
  if (int rc = fft_c2c_impl<true>(ctx, H, M, 1)) return rc;
  r2c_post_kernel<false><<<grid_for(ctx, M / 2 + 1, 256), 256, 0, ctx->stream>>>(H, M, nullptr, nullptr, nullptr);
  ctx->launches++;
  CK(cudaGetLastError());
  return 0;
}

// SRTB_B200_TRANS16=0: eight-point fused last pass; SRTB_B200_PLAN_878=0: factor 2^23 as 8,8,7 instead of 8,7,8
static bool use_trans16() {
  static const bool on = [] {
    const char* e = std::getenv("SRTB_B200_TRANS16");
    return !(e && e[0] == '0');
  }();
  return on;
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
  bool launched = false;
  if constexpr (LOGL == 7 || LOGL == 8) {
    if (use_trans16()) {
      auto kern16 = fft_trans_r2c16_tma_kernel<LOGL, T>;
      constexpr int threads = 2 * T * (L / 16);
      if (int rc = persistent_grid(ctx, kern16, threads, smem, smem, ntiles, &grid)) return rc;
      grid = std::min<unsigned>(grid, 2048);
      CK(launch_pdl(ctx, kern16, dim3(grid), dim3(threads), smem, tm, out, (uint32_t)A, (uint32_t)S, (uint32_t)L1,
                    (uint32_t)tiles_per_rest, (uint32_t)ntiles, tw, ctx->partial, (uint32_t)rest_inner));
      launched = true;
    }
  }
  if (!launched && rest_inner > 1) return 0;  // four-sweep row order: sixteen-point kernel only
  if (!launched) {
    auto kern = fft_trans_r2c_tma_kernel<LOGL, T>;
    if (int rc = persistent_grid(ctx, kern, 2 * pass_threads<LOGL, T>::value, smem, smem, ntiles, &grid)) return rc;
    grid = std::min<unsigned>(grid, 2048);
    kern<<<grid, 2 * pass_threads<LOGL, T>::value, smem, ctx->stream>>>(tm, out, (uint32_t)A, (uint32_t)S, (uint32_t)L1,
                                                                        (uint32_t)tiles_per_rest, (uint32_t)ntiles, tw,
                                                                        ctx->partial);
  }
  ctx->launches++;
  CK(cudaGetLastError());
  {
    const size_t pairs = ((A << LOGL) / L1) / 2 + 1;
    const unsigned fgrid = (unsigned)std::min<size_t>((pairs + 255) / 256, 2048);
    if (grid + fgrid > 4096) return fail(ctx, SRTB_B200_E_SIZE, "r2c: partial buffer too small");
    CK(launch_pdl(ctx, r2c_col0_fixup_kernel, dim3(fgrid), dim3(256), 0, out, (size_t)(A << LOGL), (size_t)L1, ctx->partial,
                  (unsigned)grid, ctx->ticket, ctx->mean));
  }
  ctx->launches++;
  CK(cudaGetLastError());
  *done = true;
  return 0;
}

// R2C whose split pass also leaves mean(|X_k|^2, k < N/2) in ctx->mean (used by process_block:
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
    if (four_sweeps(q, d_inout) && use_trans16()) {
      int l[4];
      plan4(q, l);
      if (int rc = ensure(ctx, &ctx->fft_scratch, &ctx->fft_scratch_bytes, M * sizeof(float2))) return rc;
      float2* s = static_cast<float2*>(ctx->fft_scratch);
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
      if (int rc = ensure(ctx, &ctx->fft_scratch, &ctx->fft_scratch_bytes, M * sizeof(float2))) return rc;
      float2* s = static_cast<float2*>(ctx->fft_scratch);
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
      r2c_post_kernel<true><<<grid, 256, 0, ctx->stream>>>(H, M, ctx->partial, ctx->ticket, ctx->mean);
      ctx->launches++;
      CK(cudaGetLastError());
      return 0;
    }
  }
  if (raw && raw->base) return SRTB_B200_E_UNSUPPORTED;  // fused unpack needs the multi-pass TMA route
  if (int rc = fft_c2c_impl<true>(ctx, H, M, 1)) return rc;
  const unsigned grid = std::min<unsigned>(grid_for(ctx, M / 2 + 1, 256), 4096);
  r2c_post_kernel<true><<<grid, 256, 0, ctx->stream>>>(H, M, ctx->partial, ctx->ticket, ctx->mean);
  ctx->launches++;
  CK(cudaGetLastError());
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

extern "C" int srtb_b200_rfi_s1(srtb_b200_ctx* ctx, void* d_x, size_t count, float avg_threshold,
                                float norm_coef, const size_t* h_bin_ranges, size_t n_ranges,
                                float* d_mean_out) {
  API_LOCK(ctx);
  if (!ctx || !d_x) return fail(ctx, SRTB_B200_E_INVALID, "rfi_s1: null argument");
  if (count == 0) return fail(ctx, SRTB_B200_E_INVALID, "rfi_s1: zero count");
  if (n_ranges && !h_bin_ranges) return fail(ctx, SRTB_B200_E_INVALID, "rfi_s1: null ranges");
  CK(cudaSetDevice(ctx->device));
  stage_scope stats_(ctx, SRTB_B200_STAGE_RFI_S1, 24.0 * (double)count);
  float2* x = static_cast<float2*>(d_x);
  const unsigned grid = std::min<unsigned>(grid_for(ctx, count / 2 + 1, 256), 4096);
  power_sum_kernel<<<grid, 256, 0, ctx->stream>>>(x, count, ctx->partial, ctx->ticket, ctx->mean);
  ctx->launches++;
  CK(cudaGetLastError());
  if (d_mean_out) CK(cudaMemcpyAsync(d_mean_out, ctx->mean, sizeof(float), cudaMemcpyDeviceToDevice, ctx->stream));
  rfi_s1_apply_kernel<<<grid_for(ctx, count / 2 + 1, 256), 256, 0, ctx->stream>>>(x, count, ctx->mean, avg_threshold, norm_coef);
  ctx->launches++;
  CK(cudaGetLastError());
  for (size_t r0 = 0; r0 < n_ranges; r0 += 16) {
    bin_ranges br;
    const size_t nr = std::min<size_t>(16, n_ranges - r0);
    size_t longest = 1;
    for (size_t r = 0; r < nr; r++) {
      const size_t lo = h_bin_ranges[2 * (r0 + r)], hi = h_bin_ranges[2 * (r0 + r) + 1];
      if (!(lo <= hi && hi < count)) return fail(ctx, SRTB_B200_E_INVALID, "rfi_s1: bin range out of bounds");
      br.lo[r] = lo;
      br.hi[r] = hi;
      longest = std::max(longest, hi - lo + 1);
    }
    dim3 g(grid_for(ctx, longest, 256), (unsigned)nr);
    rfi_zero_ranges_kernel<<<g, 256, 0, ctx->stream>>>(x, br);
    ctx->launches++;
    CK(cudaGetLastError());
  }
  return 0;
}

// ------------------------------------------------------------------------------------
// dedisperse
// ------------------------------------------------------------------------------------
extern "C" int srtb_b200_dedisperse(srtb_b200_ctx* ctx, void* d_x, size_t count, float f_min, float f_c,
                                    float df, float dm) {
  API_LOCK(ctx);
  if (!ctx || !d_x) return fail(ctx, SRTB_B200_E_INVALID, "dedisperse: null argument");
  if (count == 0) return 0;
  CK(cudaSetDevice(ctx->device));
  stage_scope stats_(ctx, SRTB_B200_STAGE_DEDISPERSE, 16.0 * (double)count);
  constexpr double D = 4.148808e3;  // coherent_dedispersion.hpp:67
  const double ddm = (D * 1e6) * (double)dm;
  dedisperse_kernel<false><<<grid_for(ctx, count / 2 + 1, 256, 16), 256, 0, ctx->stream>>>(
      static_cast<const float2*>(d_x), static_cast<float2*>(d_x), count, (double)f_min, (double)df, (double)f_c, ddm, nullptr, 0.f, 1.f);
  ctx->launches++;
  CK(cudaGetLastError());
  return 0;
}

// s1 (mean -> zap/normalise) and the chirp in two kernels instead of three: power sum, then one
// fused apply + chirp sweep, then the manual zap (zero * chirp = zero, so the order is equivalent)
// mitigate_rfi_manual (rfi_mitigation.hpp:97-158): zero the listed bin ranges, 16 ranges per launch
static int zero_bin_ranges(srtb_b200_ctx* ctx, float2* x, const std::vector<size_t>& bins) {
  for (size_t r0 = 0; r0 < bins.size() / 2; r0 += 16) {
    bin_ranges br;
    const size_t nr = std::min<size_t>(16, bins.size() / 2 - r0);
    size_t longest = 1;
    for (size_t r = 0; r < nr; r++) {
      br.lo[r] = bins[2 * (r0 + r)];
      br.hi[r] = bins[2 * (r0 + r) + 1];
      longest = std::max<size_t>(longest, br.hi[r] - br.lo[r] + 1);
    }
    dim3 g(grid_for(ctx, longest, 256), (unsigned)nr);
    CK(launch_pdl(ctx, rfi_zero_ranges_kernel, g, dim3(256), 0, x, br));
    ctx->launches++;
    CK(cudaGetLastError());
  }
  return 0;
}

static int rfi_s1_dedisperse_fused(srtb_b200_ctx* ctx, float2* x, size_t count, float avg_threshold, float coef,
                                   const std::vector<size_t>& bins, float f_min, float f_c, float df, float dm,
                                   bool mean_ready, const float2* src = nullptr) {
  if (!src) src = x;  // in place unless a separate (kept) spectrum is given
  if (!mean_ready) {
    const unsigned grid = std::min<unsigned>(grid_for(ctx, count / 2 + 1, 256), 4096);
    power_sum_kernel<<<grid, 256, 0, ctx->stream>>>(x, count, ctx->partial, ctx->ticket, ctx->mean);
    ctx->launches++;
    CK(cudaGetLastError());
  }
  constexpr double D = 4.148808e3;
  const double ddm = (D * 1e6) * (double)dm;
  dedisperse_kernel<true><<<grid_for(ctx, count / 2 + 1, 256, 16), 256, 0, ctx->stream>>>(
      src, x, count, (double)f_min, (double)df, (double)f_c, ddm, ctx->mean, avg_threshold, coef);
  ctx->launches++;
  CK(cudaGetLastError());
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
extern "C" int srtb_b200_rfi_s2_sk(srtb_b200_ctx* ctx, void* d_x, size_t time_count, size_t chan_count,
                                   float sk_threshold, float* d_sk_out) {
  API_LOCK(ctx);
  if (!ctx || !d_x) return fail(ctx, SRTB_B200_E_INVALID, "rfi_s2: null argument");
  if (time_count == 0 || chan_count == 0) return fail(ctx, SRTB_B200_E_INVALID, "rfi_s2: zero size");
  CK(cudaSetDevice(ctx->device));
  stage_scope stats_(ctx, SRTB_B200_STAGE_RFI_S2, 8.0 * (double)time_count * (double)chan_count);
  const float M_ = static_cast<float>(time_count);
  float hi = sk_threshold, lo = 2 - sk_threshold;
  if (lo > hi) std::swap(lo, hi);
  const float lo_ = lo * ((M_ - 1) / (M_ + 1)) + 1, hi_ = hi * ((M_ - 1) / (M_ + 1)) + 1;
  sk_kernel<<<(unsigned)chan_count, 256, 0, ctx->stream>>>(static_cast<float2*>(d_x), time_count, lo_, hi_, d_sk_out);
  ctx->launches++;
  CK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------
// signal detect
// ------------------------------------------------------------------------------------
static int detect_prepare(srtb_b200_ctx* ctx, int slot, size_t time_count, size_t need_partial_elems) {
  const size_t series_need = (size_t)SRTB_B200_MAX_BOXCARS * time_count;
  if (ctx->series_elems < series_need) {
    if (int rc = sync_lanes(ctx)) return rc;
    for (auto& p : ctx->series) {
      if (p) CK(cudaFree(p));
      p = nullptr;
    }
    ctx->series_elems = 0;
  }
  if (!ctx->series[slot]) {
    cudaError_t e = cudaMalloc(&ctx->series[slot], series_need * sizeof(float));
    if (e != cudaSuccess) return fail(ctx, SRTB_B200_E_NOMEM, "detect: series alloc failed");
    ctx->series_elems = series_need;
  }
  {
    size_t have = ctx->acc_elems * sizeof(float);
    if (int rc = ensure(ctx, reinterpret_cast<void**>(&ctx->acc), &have, time_count * sizeof(float))) return rc;
    ctx->acc_elems = have / sizeof(float);
  }
  {
    size_t have = ctx->colsum_partial_elems * sizeof(float);
    if (int rc = ensure(ctx, reinterpret_cast<void**>(&ctx->colsum_partial), &have, need_partial_elems * sizeof(float)))
      return rc;
    ctx->colsum_partial_elems = have / sizeof(float);
  }
  return 0;
}

// column-sum reduction over `chunks` partial rows, zero count, scan, boxcar ladder
// zero_stride / zero_count_n: where the detector looks for masked channels — the first time sample of every channel
// of [C][L] (stride L, C of them; the default), or the first spectrum of [time][frequency] (stride 1; v1 detector)
static int detect_tail(srtb_b200_ctx* ctx, int slot, const float2* x, size_t time_count, size_t chan_count,
                       size_t ts_count, size_t chunks, float snr, float chan_thr, size_t max_boxcar,
                       size_t zero_stride = 0) {
  if (zero_stride == 0) zero_stride = time_count;
  float* const host_series = ctx->host_series_dst ? ctx->host_series_dst + (size_t)slot * SRTB_B200_MAX_BOXCARS * time_count : nullptr;
  stage_scope stats_(ctx, SRTB_B200_STAGE_FUSED_DETECT_TAIL, 4.0 * (double)chunks * (double)ts_count);
  CK(launch_pdl(ctx, colsum_final_scan_kernel, dim3((unsigned)std::min<size_t>((ts_count + 31) / 32, (size_t)ctx->sm_count)),
                dim3(1024), 0, (const float*)ctx->colsum_partial, ts_count, chunks, ctx->series[slot], ctx->acc, x, zero_stride,
                chan_count, chan_thr, max_boxcar, ctx->detect_ticket, ctx->d_res + slot));
  ctx->launches++;
  CK(cudaGetLastError());
  // one CTA per possible boxcar; CTAs beyond n_boxcars (known only on the device) exit at once
  unsigned max_nb = 1;
  for (size_t b = 2; b <= max_boxcar && b < ts_count && max_nb < SRTB_B200_MAX_BOXCARS; b *= 2) max_nb++;
  CK(launch_pdl(ctx, detect_boxcar_kernel, dim3(max_nb), dim3(1024), 0, ctx->series[slot], time_count, (const float*)ctx->acc,
                ts_count, snr, ctx->d_res + slot, host_series));
  ctx->launches++;
  CK(cudaGetLastError());
  ctx->slot_time_count[slot] = time_count;
  return 0;
}

static int detect_enqueue(srtb_b200_ctx* ctx, int slot, const float2* x, size_t time_count,
                          size_t chan_count, size_t time_reserved_count, float snr, float chan_thr,
                          size_t max_boxcar) {
  const size_t ts_count = (time_count <= time_reserved_count) ? time_count : time_count - time_reserved_count;
  const size_t ctas_per_chunk = (ts_count + 511) / 512;
  size_t chunks = std::max<size_t>(1, (size_t)ctx->sm_count * 8 / ctas_per_chunk);
  chunks = std::min(chunks, std::min<size_t>(128, chan_count));
  const size_t rows_per_chunk = (chan_count + chunks - 1) / chunks;
  chunks = (chan_count + rows_per_chunk - 1) / rows_per_chunk;
  if (int rc = detect_prepare(ctx, slot, time_count, chunks * ts_count)) return rc;
  CK(cudaMemsetAsync(ctx->d_res + slot, 0, sizeof(detect_dev_result), ctx->stream));
  dim3 g((unsigned)ctas_per_chunk, (unsigned)chunks);
  colsum_partial_kernel<<<g, 256, 0, ctx->stream>>>(const_cast<float2*>(x), time_count, chan_count, ts_count, rows_per_chunk,
                                                    ctx->colsum_partial, nullptr);
  ctx->launches++;
  CK(cudaGetLastError());
  return detect_tail(ctx, slot, x, time_count, chan_count, ts_count, chunks, snr, chan_thr, max_boxcar);
}

// watfft (backward C2C of every channel row) with spectral kurtosis + the detector's partial column
// sums fused into its epilogue: the dynamic spectrum is written once and not read again until the
// candidate sink. Used by process_block when one CTA holds a whole row (L = 512 .. 4096).
// s1 + chirp folded into the waterfall kernel's load (process_block, L = 1024..4096): SRTB_B200_FUSE_CHIRP=0 keeps
// the separate dedisperse kernel
static bool use_fused_chirp() {
  static const bool on = [] {
    const char* e = std::getenv("SRTB_B200_FUSE_CHIRP");
    return !(e && e[0] == '0');
  }();
  return on;
}
static bool chirp_fusable(size_t time_count) {
  if (!use_fused_chirp()) return false;
  if (time_count == 8192 || time_count == 16384) return use_bigrow();
  return use_row16() && (time_count == 1024 || time_count == 2048 || time_count == 4096);
}

template <int LOGL>
static int watfft_sk_launch(srtb_b200_ctx* ctx, float2* x, size_t chan_count, float lo_, float hi_, size_t ts_count,
                            size_t* chunks_out, const row_chirp_params* chirp = nullptr, const float2* src = nullptr) {
  if (!src) src = x;  // in place unless the input spectrum is kept (DM sweep)
  if constexpr (has_row16<LOGL>::value && LOGL >= 10) {
    if (use_row16()) {
      constexpr int T16 = row16_t<LOGL>::value, threads = ((1 << LOGL) / 16) * T16;
      auto kern = chirp ? fft_row16_tma_kernel<LOGL, T16, false, true, true> : fft_row16_tma_kernel<LOGL, T16, false, true, false>;
      constexpr size_t smem = row16_smem<LOGL, T16>::bytes;
      const size_t ntiles = (chan_count + T16 - 1) / T16;
      unsigned grid = 1;
      if (int rc = persistent_grid(ctx, kern, threads, smem, smem, ntiles, &grid)) return rc;
      size_t have = ctx->colsum_partial_elems * sizeof(float);
      if (int rc = ensure(ctx, reinterpret_cast<void**>(&ctx->colsum_partial), &have, (size_t)grid * ts_count * sizeof(float)))
        return rc;
      ctx->colsum_partial_elems = have / sizeof(float);
      const float2* tw = nullptr;
      if (int rc = get_stage_twiddles(ctx, LOGL, &tw)) return rc;
      row_sk_params p{lo_, hi_, ctx->colsum_partial, (unsigned)ts_count};
      CK(launch_pdl(ctx, kern, dim3(grid), dim3(threads), smem, src, x, chan_count, tw, p, chirp ? *chirp : row_chirp_params{}));
      ctx->launches++;
      CK(cudaGetLastError());
      *chunks_out = grid;
      return 0;
    }
  }
  if (chirp || src != x) return fail(ctx, SRTB_B200_E_UNSUPPORTED, "watfft: fused chirp needs the sixteen-point row kernel");
  constexpr int T = row_t<LOGL>::value;
  auto kern = fft_row_tma_kernel<LOGL, T, false, true>;
  constexpr size_t smem = row_tma_smem<LOGL, T>::bytes;
  const size_t ntiles = (chan_count + T - 1) / T;
  unsigned grid = 1;
  if (int rc = persistent_grid(ctx, kern, pass_threads<LOGL, T>::value, smem, smem, ntiles, &grid)) return rc;
  {
    size_t have = ctx->colsum_partial_elems * sizeof(float);
    if (int rc = ensure(ctx, reinterpret_cast<void**>(&ctx->colsum_partial), &have, (size_t)grid * ts_count * sizeof(float)))
      return rc;
    ctx->colsum_partial_elems = have / sizeof(float);
  }
  const float2* tw = nullptr;
  if (int rc = get_stage_twiddles(ctx, LOGL, &tw)) return rc;
  row_sk_params p{lo_, hi_, ctx->colsum_partial, (unsigned)ts_count};
  kern<<<grid, pass_threads<LOGL, T>::value, smem, ctx->stream>>>(x, x, chan_count, tw, p);
  ctx->launches++;
  CK(cudaGetLastError());
  *chunks_out = grid;
  return 0;
}

static int watfft_sk_detect_fused(srtb_b200_ctx* ctx, int slot, float2* x, size_t time_count, size_t chan_count,
                                  size_t time_reserved_count, float sk_threshold, float snr, float chan_thr,
                                  size_t max_boxcar, const row_chirp_params* chirp = nullptr,
                                  const float2* src = nullptr) {
  const size_t ts_count = (time_count <= time_reserved_count) ? time_count : time_count - time_reserved_count;
  if (int rc = detect_prepare(ctx, slot, time_count, 1)) return rc;
  // the result header is zeroed here unless the block path did it for every stream up front (a memset between two
  // kernels would break their programmatic-dependent-launch chain)
  if (!ctx->res_zeroed) CK(cudaMemsetAsync(ctx->d_res + slot, 0, sizeof(detect_dev_result), ctx->stream));
  const float M_ = static_cast<float>(time_count);
  float hi = sk_threshold, lo = 2 - sk_threshold;
  if (lo > hi) std::swap(lo, hi);
  const float lo_ = lo * ((M_ - 1) / (M_ + 1)) + 1, hi_ = hi * ((M_ - 1) / (M_ + 1)) + 1;
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
    }
    const float2* s_ = src ? src : x;
    rc = (time_count == 8192) ? launch_bigrow<13, false>(ctx, s_, x, chan_count, &p, chirp ? &cpv : nullptr, &chunks)
                              : launch_bigrow<14, false>(ctx, s_, x, chan_count, &p, chirp ? &cpv : nullptr, &chunks);
    if (rc) return rc;
    stats_.reset();
    return detect_tail(ctx, slot, x, time_count, chan_count, ts_count, chunks, snr, chan_thr, max_boxcar);
  }
  switch (ilog2(time_count)) {
    case 9: rc = watfft_sk_launch<9>(ctx, x, chan_count, lo_, hi_, ts_count, &chunks, chirp, src); break;
    case 10: rc = watfft_sk_launch<10>(ctx, x, chan_count, lo_, hi_, ts_count, &chunks, chirp, src); break;
    case 11: rc = watfft_sk_launch<11>(ctx, x, chan_count, lo_, hi_, ts_count, &chunks, chirp, src); break;
    default: rc = watfft_sk_launch<12>(ctx, x, chan_count, lo_, hi_, ts_count, &chunks, chirp, src); break;
  }
  if (rc) return rc;
  stats_.reset();
  return detect_tail(ctx, slot, x, time_count, chan_count, ts_count, chunks, snr, chan_thr, max_boxcar);
}

// Rows longer than one CTA's shared memory (2^15 .. 2^20 time samples; the shipped configurations have 2^18):
//   sweep A  column FFTs with rfi_mitigation_s1 + the chirp applied as the tile is read  (spectrum -> scratch)
//   sweep B  transposing last sweep, leaving per-tile (sum |y|^2, sum |y|^4)              (scratch -> spectrum)
//   decide   one thread per channel folds its tiles and takes the SK decision
//   sums     the detector's partial column sums, zeroing the flagged rows on the way (one read of the spectrum)
// i.e. 20 bytes per sample instead of the 32 of dedisperse + two-sweep waterfall + SK + column sums.
static bool long_fusable(size_t time_count, const float2* x) {
  static const bool on = [] {
    const char* e = std::getenv("SRTB_B200_LONG_FUSED");
    return !(e && e[0] == '0');
  }();
  const int q = ilog2(time_count);
  return on && use_fused_chirp() && use_col16() && is_pow2(time_count) && q >= 15 && q <= 18 && get_encode_tiled() &&
         (reinterpret_cast<uintptr_t>(x) & 15u) == 0;
}

static int watfft_long_fused(srtb_b200_ctx* ctx, int slot, float2* x, const float2* src, size_t time_count,
                             size_t chan_count, size_t time_reserved_count, float sk_threshold, float snr,
                             float chan_thr, size_t max_boxcar, const row_chirp_params& chirp) {
  const size_t ts_count = (time_count <= time_reserved_count) ? time_count : time_count - time_reserved_count;
  const int q = ilog2(time_count);
  const int l1 = (q + 1) / 2, l2 = q - l1;
  const size_t L1 = (size_t)1 << l1, L2 = (size_t)1 << l2;
  if (int rc = ensure(ctx, &ctx->fft_scratch, &ctx->fft_scratch_bytes, chan_count * time_count * sizeof(float2))) return rc;
  float2* s = static_cast<float2*>(ctx->fft_scratch);
  const size_t T_last = (l2 <= 8) ? 16 : 8;  // rows per tile of the last sweep (col_t)
  const size_t tiles_per_row = L1 / T_last;
  if (int rc = ensure(ctx, &ctx->long_stats, &ctx->long_stats_bytes, chan_count * tiles_per_row * sizeof(float2))) return rc;
  if (int rc = ensure(ctx, &ctx->long_zap, &ctx->long_zap_bytes, chan_count)) return rc;
  float2* stats = static_cast<float2*>(ctx->long_stats);
  unsigned char* zap = static_cast<unsigned char*>(ctx->long_zap);
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
  const float M_ = static_cast<float>(time_count);
  float hi = sk_threshold, lo = 2 - sk_threshold;
  if (lo > hi) std::swap(lo, hi);
  const float lo_ = lo * ((M_ - 1) / (M_ + 1)) + 1, hi_ = hi * ((M_ - 1) / (M_ + 1)) + 1;
  sk_decide_kernel<<<(unsigned)((chan_count + 255) / 256), 256, 0, ctx->stream>>>(stats, (unsigned)tiles_per_row, chan_count,
                                                                             M_, lo_, hi_, zap);
  ctx->launches++;
  CK(cudaGetLastError());
  // partial column sums (all time samples are visited so that flagged rows are zeroed completely)
  const size_t ctas_per_chunk = (time_count + 511) / 512;
  size_t chunks = std::max<size_t>(1, (size_t)ctx->sm_count * 8 / ctas_per_chunk);
  chunks = std::min(chunks, std::min<size_t>(128, chan_count));
  const size_t rows_per_chunk = (chan_count + chunks - 1) / chunks;
  chunks = (chan_count + rows_per_chunk - 1) / rows_per_chunk;
  if (int rc2 = detect_prepare(ctx, slot, time_count, chunks * ts_count)) return rc2;
  if (!ctx->res_zeroed) CK(cudaMemsetAsync(ctx->d_res + slot, 0, sizeof(detect_dev_result), ctx->stream));
  dim3 g((unsigned)ctas_per_chunk, (unsigned)chunks);
  colsum_partial_kernel<<<g, 256, 0, ctx->stream>>>(x, time_count, chan_count, ts_count, rows_per_chunk, ctx->colsum_partial, zap);
  ctx->launches++;
  CK(cudaGetLastError());
  stats_.reset();
  return detect_tail(ctx, slot, x, time_count, chan_count, ts_count, chunks, snr, chan_thr, max_boxcar);
}

// s2 (spectral kurtosis) + the detector's first column-sum stage in one sweep; used by process_block
// when a row fits the per-thread register tile (L = 512 .. 4096)
static bool sk_detect_fusable(size_t time_count) {
  return time_count == 512 || time_count == 1024 || time_count == 2048 || time_count == 4096;
}
// waterfall FFT + SK + column sums in one kernel (no chirp): the row kernels above plus the whole-row kernel
static bool watfft_sk_fusable(size_t time_count) {
  return sk_detect_fusable(time_count) || ((time_count == 8192 || time_count == 16384) && use_bigrow());
}
static int sk_detect_fused(srtb_b200_ctx* ctx, int slot, float2* x, size_t time_count, size_t chan_count,
                           size_t time_reserved_count, float sk_threshold, float snr, float chan_thr,
                           size_t max_boxcar) {
  const size_t ts_count = (time_count <= time_reserved_count) ? time_count : time_count - time_reserved_count;
  const size_t rows_per_chunk = std::max<size_t>(1, chan_count / ((size_t)ctx->sm_count * 4));
  const size_t chunks = (chan_count + rows_per_chunk - 1) / rows_per_chunk;
  if (int rc = detect_prepare(ctx, slot, time_count, chunks * ts_count)) return rc;
  CK(cudaMemsetAsync(ctx->d_res + slot, 0, sizeof(detect_dev_result), ctx->stream));
  const float M_ = static_cast<float>(time_count);
  float hi = sk_threshold, lo = 2 - sk_threshold;
  if (lo > hi) std::swap(lo, hi);
  const float lo_ = lo * ((M_ - 1) / (M_ + 1)) + 1, hi_ = hi * ((M_ - 1) / (M_ + 1)) + 1;
  switch (time_count / 512) {
    case 1: sk_colsum_kernel<1><<<(unsigned)chunks, 256, 0, ctx->stream>>>(x, time_count, chan_count, ts_count, rows_per_chunk, lo_, hi_, ctx->colsum_partial); break;
    case 2: sk_colsum_kernel<2><<<(unsigned)chunks, 256, 0, ctx->stream>>>(x, time_count, chan_count, ts_count, rows_per_chunk, lo_, hi_, ctx->colsum_partial); break;
    case 4: sk_colsum_kernel<4><<<(unsigned)chunks, 256, 0, ctx->stream>>>(x, time_count, chan_count, ts_count, rows_per_chunk, lo_, hi_, ctx->colsum_partial); break;
    default: sk_colsum_kernel<8><<<(unsigned)chunks, 256, 0, ctx->stream>>>(x, time_count, chan_count, ts_count, rows_per_chunk, lo_, hi_, ctx->colsum_partial); break;
  }
  ctx->launches++;
  CK(cudaGetLastError());
  return detect_tail(ctx, slot, x, time_count, chan_count, ts_count, chunks, snr, chan_thr, max_boxcar);
}

static int detect_collect(srtb_b200_ctx* ctx, int slot, srtb_b200_detect_result* h_result, float* h_series,
                          int copy_all) {
  static_assert(sizeof(detect_dev_result) == sizeof(srtb_b200_detect_result), "result layout");
  std::memcpy(h_result, ctx->h_res + slot, sizeof(srtb_b200_detect_result));
  if (h_series && h_result->detect_enabled) {
    const size_t stride = ctx->slot_time_count[slot];
    bool any = false;
    for (int b = 0; b < h_result->n_boxcars; b++) {
      if (copy_all || h_result->signal_count[b] > 0) {
        CK(cudaMemcpyAsync(h_series + (size_t)b * stride, ctx->series[slot] + (size_t)b * stride,
                           h_result->series_length[b] * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
        any = true;
      }
    }
    if (any) CK(cudaStreamSynchronize(ctx->stream));
  } else if (h_series && copy_all) {
    // detection disabled: still hand back the mean-removed time series
    CK(cudaMemcpyAsync(h_series, ctx->series[slot], h_result->time_series_count * sizeof(float),
                       cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  return 0;
}

extern "C" int srtb_b200_signal_detect(srtb_b200_ctx* ctx, const void* d_x, size_t time_count,
                                       size_t chan_count, size_t time_reserved_count, float snr_threshold,
                                       float channel_threshold, size_t max_boxcar_length,
                                       srtb_b200_detect_result* h_result, float* h_series, int copy_all) {
  API_LOCK(ctx);
  if (!ctx || !d_x || !h_result) return fail(ctx, SRTB_B200_E_INVALID, "signal_detect: null argument");
  if (time_count == 0 || chan_count == 0) return fail(ctx, SRTB_B200_E_INVALID, "signal_detect: zero size");
  CK(cudaSetDevice(ctx->device));
  stage_scope stats_(ctx, SRTB_B200_STAGE_SIGNAL_DETECT, 8.0 * (double)time_count * (double)chan_count);
  if (int rc = detect_enqueue(ctx, 0, static_cast<const float2*>(d_x), time_count, chan_count,
                              time_reserved_count, snr_threshold, channel_threshold, max_boxcar_length))
    return rc;
  CK(cudaMemcpyAsync(ctx->h_res, ctx->d_res, sizeof(detect_dev_result), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return detect_collect(ctx, 0, h_result, h_series, copy_all);
}

// ---- alternates of the refft path: spectra laid out [time][frequency] ------------------------------------------
static int sk_v1_enqueue(srtb_b200_ctx* ctx, float2* x, size_t fft_bins, size_t time_counts, float sk_threshold,
                         float* d_sk_out) {
  if (int rc = ensure(ctx, &ctx->long_zap, &ctx->long_zap_bytes, fft_bins)) return rc;
  unsigned char* zap = static_cast<unsigned char*>(ctx->long_zap);
  const float M_ = static_cast<float>(time_counts);
  float hi = sk_threshold, lo = 2 - sk_threshold;
  if (lo > hi) std::swap(lo, hi);
  const float lo_ = lo * ((M_ - 1) / (M_ + 1)) + 1, hi_ = hi * ((M_ - 1) / (M_ + 1)) + 1;
  sk_v1_stats_kernel<<<(unsigned)((fft_bins + 31) / 32), 256, 0, ctx->stream>>>(x, fft_bins, time_counts, lo_, hi_, zap, d_sk_out);
  ctx->launches++;
  CK(cudaGetLastError());
  const unsigned gy = (unsigned)std::max<size_t>(1, std::min<size_t>(time_counts, 64));
  sk_v1_zero_kernel<<<dim3((unsigned)((fft_bins + 255) / 256), gy), 256, 0, ctx->stream>>>(x, fft_bins, time_counts, zap);
  ctx->launches++;
  CK(cudaGetLastError());
  return 0;
}

extern "C" int srtb_b200_rfi_sk_v1(srtb_b200_ctx* ctx, void* d_x, size_t fft_bins, size_t time_counts,
                                   float sk_threshold, float* d_sk_out) {
  API_LOCK(ctx);
  if (!ctx || !d_x) return fail(ctx, SRTB_B200_E_INVALID, "rfi_sk_v1: null argument");
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
  if (count_per_batch == 0 || batch_size == 0) return fail(ctx, SRTB_B200_E_INVALID, "signal_detect_v1: zero size");
  CK(cudaSetDevice(ctx->device));
  float2* x = static_cast<float2*>(d_x);
  if (int rc = sk_v1_enqueue(ctx, x, count_per_batch, batch_size, sk_threshold, nullptr)) return rc;
  // one value per spectrum; then the same tail as the v2 detector (mean removal, scan, boxcars) on a series of
  // batch_size values, masked channels counted over the first spectrum
  if (int rc = detect_prepare(ctx, 0, batch_size, batch_size)) return rc;
  CK(cudaMemsetAsync(ctx->d_res, 0, sizeof(detect_dev_result), ctx->stream));
  rowsum_norm_kernel<<<(unsigned)((batch_size + 7) / 8), 256, 0, ctx->stream>>>(x, count_per_batch, batch_size, ctx->colsum_partial);
  ctx->launches++;
  CK(cudaGetLastError());
  if (int rc = detect_tail(ctx, 0, x, batch_size, count_per_batch, batch_size, 1, snr_threshold, channel_threshold,
                           max_boxcar_length, /*zero_stride=*/1))
    return rc;
  CK(cudaMemcpyAsync(ctx->h_res, ctx->d_res, sizeof(detect_dev_result), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
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

// enqueue every stage of one block on ctx->stream (no host sync); results land in
// ctx->h_res[res_base .. res_base + streams) once the stream reaches the final D2H copy
// unpack fused into the first FFT sweep: possible when the samples are 8-bit, the window is the rectangle and every
// complex point of a stream is one fixed-size byte group (simple, "1 1 2 2", "1 2 1 2"); fills raw[stream]
static bool raw_sources_for(const srtb_b200_block_config* cfg, const void* d_baseband, size_t baseband_bytes, int streams,
                            raw_source (&raw)[4]) {
  const int bits = cfg->baseband_input_bits;
  const int fmt = cfg->baseband_format;
  const size_t N = cfg->baseband_input_count;
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

// (re)allocate one set of per-stream working buffers of N + 2 floats (the in-place buffer of the reference's works,
// unpack_pipe.hpp:65-67) owned by the ctx
static int ensure_stream_bufs(srtb_b200_ctx* ctx, float* (&bufs)[4], size_t* elems, size_t N, int streams) {
  if (*elems < N + 2) {
    if (int rc = sync_lanes(ctx)) return rc;
    for (auto& p : bufs) {
      if (p) CK(cudaFree(p));
      p = nullptr;
    }
    *elems = 0;
  }
  for (int s = 0; s < streams; s++)
    if (!bufs[s]) {
      cudaError_t e = cudaMalloc(&bufs[s], (N + 2) * sizeof(float));
      if (e != cudaSuccess) return fail(ctx, SRTB_B200_E_NOMEM, "process_block: stream buffer alloc failed");
    }
  *elems = N + 2;
  return 0;
}

// bufs[s]: working buffer of stream s (N + 2 floats, 16-byte aligned for the fused routes) — holds the dynamic
// spectrum [C][L] when the block is done. host_series (optional): pinned host memory that receives positive series.
// K12 phase table for the whole-row waterfall kernel (block path; SRTB_B200_CHIRP_TABLE=0 evaluates every phase on the
// fly like the DM sweep does). Rebuilt when the geometry or the DM changes; built synchronously, so both lanes and any
// later launch may read it.
static bool use_chirp_table() {
  static const bool on = [] {
    const char* e = std::getenv("SRTB_B200_CHIRP_TABLE");
    return !(e && e[0] == '0');
  }();
  return on;
}
static int get_chirp_table(srtb_b200_ctx* ctx, size_t n, const row_chirp_params& cp, const float** out) {
  *out = nullptr;
  if (!use_chirp_table() || n * sizeof(float) > ((size_t)4 << 30)) return 0;
  const double key[6] = {(double)n, cp.f_min, cp.df, cp.inv_fc, cp.f_c, cp.ddm};
  if (ctx->chirp_tab && std::memcmp(key, ctx->chirp_tab_key, sizeof(key)) == 0) {
    *out = ctx->chirp_tab;
    return 0;
  }
  if (int rc = ensure(ctx, reinterpret_cast<void**>(&ctx->chirp_tab), &ctx->chirp_tab_bytes, n * sizeof(float))) return rc;
  if (int rc = sync_lanes(ctx)) return rc;  // a block still in flight may be reading the previous table
  chirp_phase_table_kernel<<<grid_for(ctx, n, 256), 256, 0, ctx->stream>>>(ctx->chirp_tab, n, cp.f_min, cp.df, cp.inv_fc,
                                                                           cp.f_c, cp.ddm);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(ctx->stream));
  std::memcpy(ctx->chirp_tab_key, key, sizeof(key));
  *out = ctx->chirp_tab;
  return 0;
}

// second lane of a context (see srtb_b200_ctx::lane_state): created on first use
static int ensure_alt_lane(srtb_b200_ctx* ctx) {
  if (ctx->alt_ready) return 0;
  auto& a = ctx->alt;
  {
    // SRTB_B200_LANE_PRIORITY=1: the second lane at the lowest stream priority, so that its CTAs only fill what the
    // first lane leaves free instead of being co-scheduled with it (experiment; default: equal priorities)
    const char* e = std::getenv("SRTB_B200_LANE_PRIORITY");
    if (e && e[0] == '1') {
      int lo = 0, hi = 0;
      CK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
      CK(cudaStreamCreateWithPriority(&a.stream, cudaStreamNonBlocking, lo));
    } else {
      CK(cudaStreamCreateWithFlags(&a.stream, cudaStreamNonBlocking));
    }
  }
  CK(cudaMalloc(&a.partial, sizeof(double) * 4096));
  CK(cudaMalloc(&a.ticket, sizeof(unsigned)));
  CK(cudaMemset(a.ticket, 0, sizeof(unsigned)));
  CK(cudaMalloc(&a.detect_ticket, sizeof(unsigned)));
  CK(cudaMemset(a.detect_ticket, 0, sizeof(unsigned)));
  CK(cudaMalloc(&a.mean, sizeof(float)));
  CK(cudaEventCreateWithFlags(&ctx->lane_fork, cudaEventDisableTiming));
  CK(cudaEventCreateWithFlags(&ctx->lane_join, cudaEventDisableTiming));
  ctx->alt_ready = true;
  return 0;
}

// join_lanes: the first lane waits for the second at the end (process_block); the ring leaves the lanes free-running
// (each copies its own result headers back, *alt_used tells the caller to record a completion event on both).
static int block_enqueue(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg, const void* d_baseband,
                         size_t baseband_bytes, int res_base, int* streams_out, size_t* L_out, float* const* bufs,
                         float* host_series, bool join_lanes = true, bool* alt_used = nullptr) {
  const int streams = format_streams(cfg->baseband_format);
  if (!streams) return fail(ctx, SRTB_B200_E_UNSUPPORTED, "process_block: unknown format");
  const size_t N = cfg->baseband_input_count;
  if (N < 2 || !is_pow2(N)) return fail(ctx, SRTB_B200_E_SIZE, "[fft] n must be a power of 2, got " + std::to_string(N));
  struct series_dst_scope {  // detect_tail reads ctx->host_series_dst; it is only meaningful inside this call
    srtb_b200_ctx* c;
    ~series_dst_scope() {
      c->host_series_dst = nullptr;
      c->res_zeroed = false;
      c->pdl_auto = false;
    }
  } series_scope_{ctx};
  ctx->host_series_dst = host_series;
  ctx->pdl_auto = N <= ((size_t)1 << 25);
  // the data streams of a block are independent: odd ones go to the context's second lane (per-stage timing wants the
  // kernels alone, so it keeps one lane)
  const bool two_lanes = ctx->lanes >= 2 && streams >= 2 && !ctx->stats_on;
  if (alt_used) *alt_used = two_lanes;
  if (two_lanes) {
    if (int rc = ensure_alt_lane(ctx)) return rc;
  } else {
    // result headers zeroed before the first kernel (a memset between kernels would break the dependent-launch chain);
    // with two lanes every stream zeroes its own header at the head of its chain, on its lane
    CK(cudaMemsetAsync(ctx->d_res, 0, sizeof(detect_dev_result) * streams, ctx->stream));
  }
  ctx->res_zeroed = true;
  // unpack: fused into the first FFT pass when the samples are 8-bit and every complex point of a
  // stream is one fixed-size byte group (simple, "1 1 2 2", "1 2 1 2"); otherwise the unpack kernel
  raw_source raw[4];
  const bool fuse_unpack = raw_sources_for(cfg, d_baseband, baseband_bytes, streams, raw);
  bool unpacked = false;
  auto ensure_unpacked = [&]() -> int {
    if (unpacked) return 0;
    unpacked = true;
    return srtb_b200_unpack(ctx, d_baseband, baseband_bytes, cfg->baseband_input_bits, cfg->baseband_format,
                            cfg->window, bufs, N);
  };
  if (!fuse_unpack)
    if (int rc = ensure_unpacked()) return rc;
  const size_t Nc = N / 2;
  const size_t batch = std::min<size_t>(cfg->spectrum_channel_count, Nc);  // fft_pipe.hpp:318-320
  if (batch == 0 || !is_pow2(batch)) return fail(ctx, SRTB_B200_E_SIZE, "spectrum_channel_count must be a power of 2");
  const size_t L = Nc / batch;
  // manual zap ranges -> bins (host, rfi_mitigation.hpp:102-143)
  std::vector<size_t> bins;
  for (uint64_t r = 0; r < cfg->n_rfi_freq_pairs; r++) {
    size_t lo, hi;
    if (srtb_b200_rfi_range_to_bins(cfg->rfi_freq_pairs[2 * r], cfg->rfi_freq_pairs[2 * r + 1],
                                    cfg->baseband_freq_low, cfg->baseband_bandwidth, Nc, &lo, &hi)) {
      bins.push_back(lo);
      bins.push_back(hi);
    }
  }
  const float coef = srtb_b200_norm_coefficient(Nc, cfg->spectrum_channel_count);
  const float df = cfg->baseband_bandwidth / static_cast<float>(Nc);  // dedisperse_pipe.hpp:34
  const float f_min = cfg->baseband_freq_low, f_c = f_min + cfg->baseband_bandwidth;
  const size_t reserved = srtb_b200_nsamps_reserved(N, cfg->spectrum_channel_count, cfg->baseband_freq_low,
                                                    cfg->baseband_bandwidth, cfg->baseband_sample_rate, cfg->dm,
                                                    cfg->baseband_reserve_sample) /
                          batch;
  auto fork_lanes = [&]() -> int {  // called on the first lane: the second lane continues from this point of it
    CK(cudaEventRecord(ctx->lane_fork, ctx->stream));
    CK(cudaStreamWaitEvent(ctx->alt.stream, ctx->lane_fork, 0));
    return 0;
  };
  if (two_lanes)
    if (int rc = fork_lanes()) return rc;
  auto enqueue_stream = [&](int s) -> int {
    float* buf = bufs[s];
    if (two_lanes) CK(cudaMemsetAsync(ctx->d_res + s, 0, sizeof(detect_dev_result), ctx->stream));
    {
      stage_scope stats_(ctx, SRTB_B200_STAGE_FUSED_R2C,
                         (double)N * (fuse_unpack ? (double)std::abs(cfg->baseband_input_bits) / 8.0 : 4.0) + 4.0 * (double)N);
      int rc = SRTB_B200_E_UNSUPPORTED;
      if (fuse_unpack && !unpacked) rc = fft_r2c_with_power_mean(ctx, buf, N, &raw[s], nullptr);
      if (rc == SRTB_B200_E_UNSUPPORTED) {
        // this size/alignment cannot take the fused route: unpack all streams once, then the plain R2C. The route is a
        // property of the block (same size and base pointer for every stream), so it can only change on stream 0;
        // later it would overwrite finished streams with their unpacked input
        if (fuse_unpack && !unpacked && s > 0)
          return fail(ctx, SRTB_B200_E_UNSUPPORTED, "process_block: fused unpack refused stream " + std::to_string(s) + " after accepting stream 0");
        const bool was_unpacked = unpacked;
        if (int rc2 = ensure_unpacked()) return rc2;
        if (two_lanes && !was_unpacked)
          if (int rc2 = fork_lanes()) return rc2;  // s == 0 here: the second lane must see the unpacked samples
        rc = fft_r2c_with_power_mean(ctx, buf, N);
      }
      if (rc) return rc;
    }
    const bool aligned = (reinterpret_cast<uintptr_t>(buf) & 15u) == 0;
    if (chirp_fusable(L) && aligned) {
      // manual zap on the raw spectrum (0 stays 0 through s1 and the chirp), then ONE kernel: s1 + chirp on load,
      // waterfall FFT, SK, partial column sums
      if (int rc = zero_bin_ranges(ctx, reinterpret_cast<float2*>(buf), bins)) return rc;
      constexpr double D = 4.148808e3;  // coherent_dedispersion.hpp:67
      row_chirp_params cp{(double)f_min, (double)df, 1.0 / (double)f_c, (double)f_c, (D * 1e6) * (double)cfg->dm,
                          ctx->mean, cfg->mitigate_rfi_average_method_threshold, coef};
      if (int rc = get_chirp_table(ctx, Nc, cp, &cp.phase)) return rc;
      if (int rc = watfft_sk_detect_fused(ctx, s, reinterpret_cast<float2*>(buf), L, batch, reserved,
                                          cfg->mitigate_rfi_spectral_kurtosis_threshold,
                                          cfg->signal_detect_signal_noise_threshold,
                                          cfg->signal_detect_channel_threshold, cfg->signal_detect_max_boxcar_length,
                                          &cp))
        return rc;
      return 0;
    }
    if (long_fusable(L, reinterpret_cast<float2*>(buf))) {
      // long rows: manual zap on the raw spectrum, then chirp-on-load column sweep, last sweep with SK statistics,
      // decision, column sums (20 bytes per sample)
      if (int rc = zero_bin_ranges(ctx, reinterpret_cast<float2*>(buf), bins)) return rc;
      constexpr double D = 4.148808e3;
      row_chirp_params cp{(double)f_min, (double)df, 1.0 / (double)f_c, (double)f_c, (D * 1e6) * (double)cfg->dm,
                          ctx->mean, cfg->mitigate_rfi_average_method_threshold, coef, 0};
      // (no phase table here: the long-row column sweep is DRAM-bound, and the 4 extra bytes per bin a table costs
      // outweigh the fp64 evaluation it would replace)
      const int rc = watfft_long_fused(ctx, s, reinterpret_cast<float2*>(buf), reinterpret_cast<const float2*>(buf), L, batch,
                                       reserved, cfg->mitigate_rfi_spectral_kurtosis_threshold,
                                       cfg->signal_detect_signal_noise_threshold, cfg->signal_detect_channel_threshold,
                                       cfg->signal_detect_max_boxcar_length, cp);
      if (rc != SRTB_B200_E_UNSUPPORTED) {
        if (rc) return rc;
        return 0;
      }
    }
    if (int rc = rfi_s1_dedisperse_fused(ctx, reinterpret_cast<float2*>(buf), Nc,
                                         cfg->mitigate_rfi_average_method_threshold, coef, bins, f_min, f_c, df, cfg->dm,
                                         /*mean_ready=*/true))
      return rc;
    if (watfft_sk_fusable(L) && aligned) {
      // waterfall FFT + SK + partial column sums in one kernel, then the small detector tail
      if (int rc = watfft_sk_detect_fused(ctx, s, reinterpret_cast<float2*>(buf), L, batch, reserved,
                                          cfg->mitigate_rfi_spectral_kurtosis_threshold,
                                          cfg->signal_detect_signal_noise_threshold,
                                          cfg->signal_detect_channel_threshold, cfg->signal_detect_max_boxcar_length))
        return rc;
      return 0;
    }
    if (int rc = srtb_b200_watfft_c2c_backward(ctx, buf, L, batch)) return rc;
    if (sk_detect_fusable(L)) {
      if (int rc = sk_detect_fused(ctx, s, reinterpret_cast<float2*>(buf), L, batch, reserved,
                                   cfg->mitigate_rfi_spectral_kurtosis_threshold,
                                   cfg->signal_detect_signal_noise_threshold, cfg->signal_detect_channel_threshold,
                                   cfg->signal_detect_max_boxcar_length))
        return rc;
    } else {
      if (int rc = srtb_b200_rfi_s2_sk(ctx, buf, L, batch, cfg->mitigate_rfi_spectral_kurtosis_threshold, nullptr)) return rc;
      if (int rc = detect_enqueue(ctx, s, reinterpret_cast<const float2*>(buf), L, batch, reserved,
                                  cfg->signal_detect_signal_noise_threshold, cfg->signal_detect_channel_threshold,
                                  cfg->signal_detect_max_boxcar_length))
        return rc;
    }
    return 0;
  };
  for (int s = 0; s < streams; s++) {
    const bool alt = two_lanes && (s & 1);
    if (alt) lane_swap(ctx);
    int rc = enqueue_stream(s);
    if (!rc && two_lanes) {
      const cudaError_t e = cudaMemcpyAsync(ctx->h_res + res_base + s, ctx->d_res + s, sizeof(detect_dev_result),
                                            cudaMemcpyDeviceToHost, ctx->stream);
      if (e != cudaSuccess) rc = fail(ctx, SRTB_B200_E_CUDA, std::string("result header copy: ") + cudaGetErrorString(e));
    }
    if (alt) lane_swap(ctx);
    if (rc) return rc;
  }
  if (two_lanes) {
    if (join_lanes) {
      CK(cudaEventRecord(ctx->lane_join, ctx->alt.stream));
      CK(cudaStreamWaitEvent(ctx->stream, ctx->lane_join, 0));
    }
  } else {
    CK(cudaMemcpyAsync(ctx->h_res + res_base, ctx->d_res, sizeof(detect_dev_result) * streams, cudaMemcpyDeviceToHost,
                       ctx->stream));
  }
  *streams_out = streams;
  *L_out = L;
  return 0;
}

extern "C" int srtb_b200_process_block_device(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg,
                                              const void* d_baseband, size_t baseband_bytes,
                                              srtb_b200_detect_result* h_results, float* h_series,
                                              int copy_all) {
  API_LOCK(ctx);
  if (!ctx || !cfg || !d_baseband || !h_results) return fail(ctx, SRTB_B200_E_INVALID, "process_block: null argument");
  CK(cudaSetDevice(ctx->device));
  int streams = 0;
  size_t L = 0;
  if (format_streams(cfg->baseband_format) && cfg->baseband_input_count >= 2)
    if (int rc = ensure_stream_bufs(ctx, ctx->stream_buf, &ctx->stream_buf_elems, cfg->baseband_input_count,
                                    format_streams(cfg->baseband_format)))
      return rc;
  if (int rc = block_enqueue(ctx, cfg, d_baseband, baseband_bytes, 0, &streams, &L, ctx->stream_buf, nullptr)) return rc;
  CK(cudaStreamSynchronize(ctx->stream));
  for (int s = 0; s < streams; s++)
    if (int rc = detect_collect(ctx, s, h_results + s, h_series ? h_series + (size_t)s * SRTB_B200_MAX_BOXCARS * L : nullptr, copy_all))
      return rc;
  return streams;
}

extern "C" int srtb_b200_process_block(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg,
                                       const void* h_baseband, size_t baseband_bytes,
                                       srtb_b200_detect_result* h_results, float* h_series, int copy_all) {
  API_LOCK(ctx);
  if (!ctx || !cfg || !h_baseband) return fail(ctx, SRTB_B200_E_INVALID, "process_block: null argument");
  CK(cudaSetDevice(ctx->device));
  if (int rc = ensure(ctx, &ctx->d_baseband, &ctx->d_baseband_bytes, baseband_bytes)) return rc;
  CK(cudaMemcpyAsync(ctx->d_baseband, h_baseband, baseband_bytes, cudaMemcpyHostToDevice, ctx->stream));
  return srtb_b200_process_block_device(ctx, cfg, ctx->d_baseband, baseband_bytes, h_results, h_series, copy_all);
}

// ---- DM sweep on one block (BASELINE config #4): unpack + R2C + mean once per stream, then for every
// trial DM the s1-apply + chirp (out of place, the spectrum is kept), waterfall FFT, SK and detector.
// Each trial's result equals process_block with cfg->dm = that DM on the same block.
extern "C" int srtb_b200_process_block_dm_sweep(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg,
                                                const void* baseband, size_t baseband_bytes, int on_device,
                                                const float* h_dms, size_t n_dm,
                                                srtb_b200_detect_result* h_results /* [n_dm][streams] */) {
  API_LOCK(ctx);
  if (!ctx || !cfg || !baseband || !h_dms || !h_results || n_dm == 0)
    return fail(ctx, SRTB_B200_E_INVALID, "dm_sweep: bad argument");
  CK(cudaSetDevice(ctx->device));
  const int streams = format_streams(cfg->baseband_format);
  if (!streams) return fail(ctx, SRTB_B200_E_UNSUPPORTED, "dm_sweep: unknown format");
  const size_t N = cfg->baseband_input_count;
  if (N < 2 || !is_pow2(N)) return fail(ctx, SRTB_B200_E_SIZE, "[fft] n must be a power of 2, got " + std::to_string(N));
  const void* d_baseband = baseband;
  if (!on_device) {
    if (int rc = ensure(ctx, &ctx->d_baseband, &ctx->d_baseband_bytes, baseband_bytes)) return rc;
    CK(cudaMemcpyAsync(ctx->d_baseband, baseband, baseband_bytes, cudaMemcpyHostToDevice, ctx->stream));
    d_baseband = ctx->d_baseband;
  }
  if (int rc = ensure_stream_bufs(ctx, ctx->stream_buf, &ctx->stream_buf_elems, N, streams)) return rc;
  const size_t Nc = N / 2;
  const size_t batch = std::min<size_t>(cfg->spectrum_channel_count, Nc);
  if (batch == 0 || !is_pow2(batch)) return fail(ctx, SRTB_B200_E_SIZE, "spectrum_channel_count must be a power of 2");
  const size_t L = Nc / batch;
  if (int rc = ensure(ctx, &ctx->sweep_buf, &ctx->sweep_buf_bytes, (Nc + 1) * sizeof(float2))) return rc;
  float2* W = static_cast<float2*>(ctx->sweep_buf);
  // unpack: fused into the first R2C sweep when the format allows (as in process_block), else the unpack kernel
  raw_source raw[4];
  bool fuse_unpack = raw_sources_for(cfg, d_baseband, baseband_bytes, streams, raw);
  bool unpacked = false;
  auto ensure_unpacked = [&]() -> int {
    if (unpacked) return 0;
    unpacked = true;
    return srtb_b200_unpack(ctx, d_baseband, baseband_bytes, cfg->baseband_input_bits, cfg->baseband_format,
                            cfg->window, ctx->stream_buf, N);
  };
  if (!fuse_unpack)
    if (int rc = ensure_unpacked()) return rc;
  std::vector<size_t> bins;
  for (uint64_t r = 0; r < cfg->n_rfi_freq_pairs; r++) {
    size_t lo, hi;
    if (srtb_b200_rfi_range_to_bins(cfg->rfi_freq_pairs[2 * r], cfg->rfi_freq_pairs[2 * r + 1],
                                    cfg->baseband_freq_low, cfg->baseband_bandwidth, Nc, &lo, &hi)) {
      bins.push_back(lo);
      bins.push_back(hi);
    }
  }
  const float coef = srtb_b200_norm_coefficient(Nc, cfg->spectrum_channel_count);
  const float df = cfg->baseband_bandwidth / static_cast<float>(Nc);
  const float f_min = cfg->baseband_freq_low, f_c = f_min + cfg->baseband_bandwidth;
  // every trial's result header is parked on the device and fetched once at the end: no host sync per trial
  if (int rc = ensure(ctx, &ctx->sweep_res, &ctx->sweep_res_bytes, n_dm * streams * sizeof(detect_dev_result))) return rc;
  detect_dev_result* d_sweep = static_cast<detect_dev_result*>(ctx->sweep_res);
  const bool fuse_chirp = chirp_fusable(L);
  for (int s = 0; s < streams; s++) {
    float* buf = ctx->stream_buf[s];
    {
      int rc = SRTB_B200_E_UNSUPPORTED;
      if (fuse_unpack && !unpacked) rc = fft_r2c_with_power_mean(ctx, buf, N, &raw[s], nullptr);
      if (rc == SRTB_B200_E_UNSUPPORTED) {
        if (fuse_unpack && !unpacked && s > 0) return fail(ctx, SRTB_B200_E_UNSUPPORTED, "dm_sweep: fused unpack refused a later stream");
        if (int rc2 = ensure_unpacked()) return rc2;
        rc = fft_r2c_with_power_mean(ctx, buf, N);  // leaves mean(|X|^2) in ctx->mean
      }
      if (rc) return rc;
    }
    const bool longf = long_fusable(L, W) && (reinterpret_cast<uintptr_t>(buf) & 15u) == 0;
    const bool fused = (fuse_chirp || longf) && (reinterpret_cast<uintptr_t>(buf) & 15u) == 0;
    if (fused)  // the manual zap does not depend on the DM: once, on the kept spectrum
      if (int rc = zero_bin_ranges(ctx, reinterpret_cast<float2*>(buf), bins)) return rc;
    for (size_t j = 0; j < n_dm; j++) {
      const size_t reserved = srtb_b200_nsamps_reserved(N, cfg->spectrum_channel_count, cfg->baseband_freq_low,
                                                        cfg->baseband_bandwidth, cfg->baseband_sample_rate, h_dms[j],
                                                        cfg->baseband_reserve_sample) / batch;
      if (longf) {
        constexpr double D = 4.148808e3;
        row_chirp_params cp{(double)f_min, (double)df, 1.0 / (double)f_c, (double)f_c, (D * 1e6) * (double)h_dms[j],
                            ctx->mean, cfg->mitigate_rfi_average_method_threshold, coef, 0};
        if (int rc = watfft_long_fused(ctx, 0, W, reinterpret_cast<const float2*>(buf), L, batch, reserved,
                                       cfg->mitigate_rfi_spectral_kurtosis_threshold,
                                       cfg->signal_detect_signal_noise_threshold, cfg->signal_detect_channel_threshold,
                                       cfg->signal_detect_max_boxcar_length, cp))
          return rc;
      } else if (fused) {
        constexpr double D = 4.148808e3;
        row_chirp_params cp{(double)f_min, (double)df, 1.0 / (double)f_c, (double)f_c, (D * 1e6) * (double)h_dms[j],
                            ctx->mean, cfg->mitigate_rfi_average_method_threshold, coef};
        if (int rc = watfft_sk_detect_fused(ctx, 0, W, L, batch, reserved, cfg->mitigate_rfi_spectral_kurtosis_threshold,
                                            cfg->signal_detect_signal_noise_threshold,
                                            cfg->signal_detect_channel_threshold, cfg->signal_detect_max_boxcar_length,
                                            &cp, reinterpret_cast<const float2*>(buf)))
          return rc;
      } else {
        if (int rc = rfi_s1_dedisperse_fused(ctx, W, Nc, cfg->mitigate_rfi_average_method_threshold, coef, bins, f_min,
                                             f_c, df, h_dms[j], /*mean_ready=*/true, reinterpret_cast<const float2*>(buf)))
          return rc;
        if (watfft_sk_fusable(L)) {
          if (int rc = watfft_sk_detect_fused(ctx, 0, W, L, batch, reserved, cfg->mitigate_rfi_spectral_kurtosis_threshold,
                                              cfg->signal_detect_signal_noise_threshold,
                                              cfg->signal_detect_channel_threshold, cfg->signal_detect_max_boxcar_length))
            return rc;
        } else {
          if (int rc = srtb_b200_watfft_c2c_backward(ctx, W, L, batch)) return rc;
          if (int rc = srtb_b200_rfi_s2_sk(ctx, W, L, batch, cfg->mitigate_rfi_spectral_kurtosis_threshold, nullptr)) return rc;
          if (int rc = detect_enqueue(ctx, 0, W, L, batch, reserved, cfg->signal_detect_signal_noise_threshold,
                                      cfg->signal_detect_channel_threshold, cfg->signal_detect_max_boxcar_length))
            return rc;
        }
      }
      CK(cudaMemcpyAsync(d_sweep + j * streams + s, ctx->d_res, sizeof(detect_dev_result), cudaMemcpyDeviceToDevice,
                         ctx->stream));
    }
  }
  static_assert(sizeof(detect_dev_result) == sizeof(srtb_b200_detect_result), "result layout");
  CK(cudaMemcpyAsync(h_results, d_sweep, n_dm * streams * sizeof(detect_dev_result), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return streams;
}

// tickets wrap at a multiple of the slot count, so ticket % SRTB_B200_RING_SLOTS is always the slot that was used
static inline int ring_ticket(uint64_t submit_count) {
  return (int)(submit_count % ((uint64_t)SRTB_B200_RING_SLOTS << 28));
}
extern "C" int srtb_b200_debug_set_submit_count(srtb_b200_ctx* ctx, uint64_t value) {
  API_LOCK(ctx);
  if (!ctx) return fail(nullptr, SRTB_B200_E_INVALID, "debug_set_submit_count: ctx is null");
  for (int i = 0; i < SRTB_B200_RING_SLOTS; i++)
    if (ctx->slot_busy[i]) return fail(ctx, SRTB_B200_E_INVALID, "debug_set_submit_count: ring not empty");
  ctx->submit_count = value;
  return 0;
}

// ---- pipelined ingest: the pinned-host ring of SURVEY section 8e -------------------------------
// submit() copies block k on a dedicated copy stream while block k-1 computes; collect() waits for
// one block's results. Up to SRTB_B200_RING_SLOTS blocks may be in flight.
extern "C" int srtb_b200_submit_block_ex(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg, const void* baseband,
                                         size_t baseband_bytes, int on_device, const srtb_b200_block_outputs* outputs) {
  API_LOCK(ctx);
  if (!ctx || !cfg || !baseband) return fail(ctx, SRTB_B200_E_INVALID, "submit_block: null argument");
  CK(cudaSetDevice(ctx->device));
  const int slot = (int)(ctx->submit_count % SRTB_B200_RING_SLOTS);
  if (ctx->slot_busy[slot]) return fail(ctx, SRTB_B200_E_INVALID, "submit_block: ring full, collect a block first");
  const int streams = format_streams(cfg->baseband_format);
  if (!streams) return fail(ctx, SRTB_B200_E_UNSUPPORTED, "process_block: unknown format");
  const size_t N = cfg->baseband_input_count;
  if (N < 2 || !is_pow2(N)) return fail(ctx, SRTB_B200_E_SIZE, "[fft] n must be a power of 2, got " + std::to_string(N));
  if (!ctx->slot_done[slot])
    for (int i = 0; i < SRTB_B200_RING_SLOTS; i++)
      if (!ctx->slot_done[i]) CK(cudaEventCreateWithFlags(&ctx->slot_done[i], cudaEventDisableTiming));
  // outputs: the caller's buffers (the work's own buffer, as in the reference) or this slot's ctx-owned ones
  float* bufs[4] = {nullptr, nullptr, nullptr, nullptr};
  bool user_spec = outputs && outputs->d_spectrum[0];
  if (user_spec) {
    for (int s = 0; s < streams; s++) {
      if (!outputs->d_spectrum[s]) return fail(ctx, SRTB_B200_E_INVALID, "submit_block: d_spectrum given for some streams only");
      bufs[s] = outputs->d_spectrum[s];
    }
  } else {
    if (int rc = ensure_stream_bufs(ctx, ctx->slot_stream_buf[slot], &ctx->slot_stream_elems[slot], N, streams)) return rc;
    for (int s = 0; s < streams; s++) bufs[s] = ctx->slot_stream_buf[slot][s];
  }
  const size_t Nc = N / 2;
  const size_t batch = std::min<size_t>(cfg->spectrum_channel_count ? cfg->spectrum_channel_count : 1, Nc);
  const size_t L = Nc / batch;
  float* h_series = outputs ? outputs->h_series : nullptr;
  if (!h_series) {
    const size_t need = (size_t)streams * SRTB_B200_MAX_BOXCARS * L;
    if (ctx->slot_h_series_elems[slot] < need) {
      if (int rc = sync_lanes(ctx)) return rc;
      if (ctx->slot_h_series[slot]) CK(cudaFreeHost(ctx->slot_h_series[slot]));
      ctx->slot_h_series[slot] = nullptr;
      ctx->slot_h_series_elems[slot] = 0;
      if (cudaMallocHost(&ctx->slot_h_series[slot], need * sizeof(float)) != cudaSuccess)
        return fail(ctx, SRTB_B200_E_NOMEM, "submit_block: pinned series buffer alloc failed");
      ctx->slot_h_series_elems[slot] = need;
    }
    h_series = ctx->slot_h_series[slot];
  }
  const void* d_baseband = baseband;
  if (!on_device) {
    if (!ctx->copy_stream) {
      CK(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
      for (int i = 0; i < SRTB_B200_RING_SLOTS; i++) CK(cudaEventCreateWithFlags(&ctx->slot_h2d[i], cudaEventDisableTiming));
    }
    if (int rc = ensure(ctx, &ctx->slot_baseband[slot], &ctx->slot_baseband_bytes[slot], baseband_bytes)) return rc;
    CK(cudaMemcpyAsync(ctx->slot_baseband[slot], baseband, baseband_bytes, cudaMemcpyHostToDevice, ctx->copy_stream));
    CK(cudaEventRecord(ctx->slot_h2d[slot], ctx->copy_stream));
    CK(cudaStreamWaitEvent(ctx->stream, ctx->slot_h2d[slot], 0));
    d_baseband = ctx->slot_baseband[slot];
  }
  bool alt_used = false;
  if (int rc = block_enqueue(ctx, cfg, d_baseband, baseband_bytes, 4 * (1 + slot), &ctx->slot_streams[slot],
                             &ctx->slot_L[slot], bufs, h_series, /*join_lanes=*/false, &alt_used))
    return rc;
  CK(cudaEventRecord(ctx->slot_done[slot], ctx->stream));
  ctx->slot_alt_used[slot] = alt_used;
  if (alt_used) {
    if (!ctx->slot_done_alt[slot]) CK(cudaEventCreateWithFlags(&ctx->slot_done_alt[slot], cudaEventDisableTiming));
    CK(cudaEventRecord(ctx->slot_done_alt[slot], ctx->alt.stream));
  }
  for (int s = 0; s < 4; s++) ctx->slot_out_spectrum[slot][s] = bufs[s];
  ctx->slot_out_series[slot] = h_series;
  ctx->slot_busy[slot] = true;
  const int ticket = ring_ticket(ctx->submit_count);
  ctx->slot_ticket[slot] = ticket;
  ctx->submit_count++;
  return ticket;
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

extern "C" int srtb_b200_collect_block_ex(srtb_b200_ctx* ctx, int ticket, srtb_b200_detect_result* h_results,
                                          const float** h_series, const void** d_spectrum) {
  API_LOCK(ctx);
  if (!ctx || !h_results || ticket < 0) return fail(ctx, SRTB_B200_E_INVALID, "collect_block: bad argument");
  const int slot = ticket % SRTB_B200_RING_SLOTS;
  if (!ctx->slot_busy[slot] || ctx->slot_ticket[slot] != ticket)
    return fail(ctx, SRTB_B200_E_INVALID, "collect_block: nothing submitted under this ticket");
  CK(cudaSetDevice(ctx->device));
  {
    const cudaEvent_t e0 = ctx->slot_done[slot], e1 = ctx->slot_alt_used[slot] ? ctx->slot_done_alt[slot] : nullptr;
    api_lock_.unlock();  // the wait runs unlocked (a ticket is collected once, by one thread)
    CK(cudaEventSynchronize(e0));
    if (e1) CK(cudaEventSynchronize(e1));
    api_lock_.lock();
  }
  const int streams = ctx->slot_streams[slot];
  std::memcpy(h_results, ctx->h_res + 4 * (1 + slot), sizeof(srtb_b200_detect_result) * streams);
  if (h_series) *h_series = ctx->slot_out_series[slot];
  if (d_spectrum)
    for (int s = 0; s < 4; s++) d_spectrum[s] = s < streams ? ctx->slot_out_spectrum[slot][s] : nullptr;
  ctx->slot_busy[slot] = false;
  return streams;
}

extern "C" int srtb_b200_collect_block(srtb_b200_ctx* ctx, int ticket, srtb_b200_detect_result* h_results) {
  return srtb_b200_collect_block_ex(ctx, ticket, h_results, nullptr, nullptr);
}

extern "C" const void* srtb_b200_block_spectrum(const srtb_b200_ctx* ctx, int stream) {
  if (!ctx || stream < 0 || stream >= 4) return nullptr;
  return ctx->stream_buf[stream];
}
