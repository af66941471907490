// srtb/pipeline/baseband_chain_pipe.hpp — the whole device chain as ONE pipe (SURVEY §8 f-4: the fused
// composites behind the pipe API). Stands where main.cpp:170-204 chains copy_to_device -> unpack -> fft_1d_r2c ->
// rfi_mitigation_s1 -> dedisperse -> watfft_1d_c2c -> rfi_mitigation_s2 -> signal_detect_pipe_2: takes the
// copy_to_device_work a source pipe produced (pinned host block) and returns one write_signal_work per data stream,
// the same objects signal_detect_pipe_2 hands to write_signal_pipe. Inside it is one
// srtb_b200_submit_block_ex / collect_block_ex pair per block, i.e. the fused kernels (unpack in the first FFT
// sweep, R2C split + power sum in the last, s1 + chirp + waterfall FFT + SK + column sums in one kernel), one H2D,
// one 1 KiB D2H per stream, and the positive boxcar series written to pinned host memory by the detector kernel.
// Throughput across blocks: start several of these pipes on their own cuda_queue (one CUDA stream + context each)
// popping from one MPMC work queue — blocks then alternate over contexts and overlap on the GPU.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <optional>
#include <stop_token>
#include <string>
#include <vector>

#include "srtb/config.hpp"
#include "srtb/cuda_queue.hpp"
#include "srtb/log.hpp"
#include "srtb/memory.hpp"
#include "srtb/pipeline/fold_pipe.hpp"            // fold_block_step
#include "srtb/pipeline/rfi_mitigation_pipe.hpp"  // srtb::spectrum::eval_rfi_ranges
#include "srtb/pipeline/unpack_pipe.hpp"          // resolve_format_alias
#include "srtb/program_options.hpp"               // parse_dm_list
#include "srtb/work.hpp"

namespace srtb {
namespace pipeline {

/** the subset of srtb::config the device path reads, as the C ABI wants it (config.hpp:80-249) */
struct block_config_holder {
  srtb_b200_block_config cfg{};
  std::vector<float> rfi_pairs;

  static int format_of(std::string_view name, int bits) {
    name = resolve_format_alias(name);
    if (name == "simple" || name == "fastmb_roach2") return SRTB_B200_FORMAT_SIMPLE;  // one stream (unpack_pipe.hpp:396)
    if (name == "interleaved_samples_2") return SRTB_B200_FORMAT_INTERLEAVED_2;
    if (name == "naocpsr_snap1") return bits == -8 ? SRTB_B200_FORMAT_NAOCPSR_SNAP1 : SRTB_B200_FORMAT_INTERLEAVED_2;
    if (name == "gznupsr_a1") return SRTB_B200_FORMAT_GZNUPSR_A1_2;
    if (name == "gznupsr_a1_4") return SRTB_B200_FORMAT_GZNUPSR_A1_4;
    throw std::invalid_argument("[start_unpack_pipe] Unknown format name: " + std::string{name});
  }
  static int stream_count(int format) {
    return format == SRTB_B200_FORMAT_SIMPLE ? 1 : (format == SRTB_B200_FORMAT_GZNUPSR_A1_4 ? 4 : 2);
  }

  /** re-read srtb::config (the reference's pipes read it on every call) */
  void refresh() {
    const auto& c = srtb::config;
    cfg.baseband_input_count = c.baseband_input_count;
    cfg.baseband_input_bits = c.baseband_input_bits;
    cfg.baseband_format = format_of(c.baseband_format_type, c.baseband_input_bits);
    cfg.window = SRTB_B200_WINDOW_RECTANGLE;  // default_window, fft_window.hpp:83
    cfg.baseband_reserve_sample = c.baseband_reserve_sample ? 1 : 0;
    cfg.baseband_freq_low = static_cast<float>(c.baseband_freq_low);
    cfg.baseband_bandwidth = static_cast<float>(c.baseband_bandwidth);
    cfg.baseband_sample_rate = static_cast<float>(c.baseband_sample_rate);
    cfg.dm = static_cast<float>(c.dm);
    cfg.mitigate_rfi_average_method_threshold = static_cast<float>(c.mitigate_rfi_average_method_threshold);
    cfg.mitigate_rfi_spectral_kurtosis_threshold = static_cast<float>(c.mitigate_rfi_spectral_kurtosis_threshold);
    cfg.spectrum_channel_count = c.spectrum_channel_count;
    cfg.signal_detect_signal_noise_threshold = static_cast<float>(c.signal_detect_signal_noise_threshold);
    cfg.signal_detect_channel_threshold = static_cast<float>(c.signal_detect_channel_threshold);
    cfg.signal_detect_max_boxcar_length = c.signal_detect_max_boxcar_length;
    cfg.signal_detect_sum_streams = c.signal_detect_sum_polarizations ? 1 : 0;
    rfi_pairs.clear();
    for (const auto& r : srtb::spectrum::eval_rfi_ranges(c.mitigate_rfi_freq_list)) {
      rfi_pairs.push_back(r.first);
      rfi_pairs.push_back(r.second);
    }
    cfg.rfi_freq_pairs = rfi_pairs.data();
    cfg.n_rfi_freq_pairs = rfi_pairs.size() / 2;
  }
};

/** the host series of stream s's positive boxcars: views into the pinned [streams][MAX_BOXCARS][L] buffer h_series,
 *  which they keep alive. row_stride: the distance between a stream's boxcar rows (0 = L; the incoherent search writes
 *  rows of T <= L) */
inline std::vector<srtb::work::time_series_holder> positive_series(const srtb_b200_detect_result& res,
                                                                   const std::shared_ptr<srtb::real>& h_series, int s,
                                                                   size_t L, size_t row_stride = 0) {
  std::vector<srtb::work::time_series_holder> out;
  srtb::real* base = h_series.get() + (size_t)s * SRTB_B200_MAX_BOXCARS * L;
  if (row_stride == 0) row_stride = L;
  for (int b = 0; b < res.n_boxcars; b++) {
    if (res.signal_count[b] == 0) continue;
    srtb::work::time_series_holder h;
    h.time_series_length = res.series_length[b];
    h.boxcar_length = res.boxcar_length[b];
    h.signal_count = res.signal_count[b];
    h.h_time_series = std::shared_ptr<srtb::real>(h_series, base + (size_t)b * row_stride);
    out.push_back(h);
  }
  return out;
}

/** one summary per trial of stream s: results and peaks are [n_dm][stride] (stride: the DM sweep's streams, 1 for the
 *  incoherent search) */
inline std::vector<srtb::work::dm_trial_summary> dm_trials(const srtb_b200_detect_result* results,
                                                           const srtb_b200_peak* peaks,
                                                           const std::vector<srtb::real>& dms, size_t stride, int s) {
  std::vector<srtb::work::dm_trial_summary> out;
  for (size_t j = 0; j < dms.size(); j++) {
    const srtb_b200_detect_result& t = results[j * stride + s];
    const srtb_b200_peak& pk = peaks[j * stride + s];
    srtb::work::dm_trial_summary d;
    d.dm = dms[j];
    d.detect_enabled = t.detect_enabled != 0;
    for (int b = 0; b < t.n_boxcars; b++)
      d.boxcars.push_back({t.boxcar_length[b], t.series_length[b], t.signal_count[b], t.threshold[b], pk.snr[b],
                           pk.peak_index[b]});
    out.push_back(std::move(d));
  }
  return out;
}

/** the block's own share of candidate windows (series indices): min(step, valid_samples) / 2C, step = fold_block_step(),
 *  or step / 2C for a block without a first_sample (UDP). Consecutive blocks start step samples apart, so a pulse in the
 *  coherent sweep's overlap is listed by one block only; the incoherent search's series are step / 2C long, so it keeps
 *  every candidate. A representative within a few samples of the boundary may be chosen differently by the two blocks */
inline uint64_t candidate_share(const srtb::work::write_signal_work& w) {
  const uint64_t two_c = 2 * (uint64_t)w.batch_size, step = fold_block_step();
  if (two_c == 0) return 0;
  return (w.first_sample != w.no_first_sample ? std::min(step, w.valid_samples) : step) / two_c;
}

/** events (at most cap of the true total n_events) clustered into out; a warning names both counts, and `who`, when the
 *  cap cut the list */
inline void cluster_candidates(std::vector<srtb::work::dm_candidate>& out, const srtb_b200_event* events,
                               uint64_t n_events, size_t cap, const std::vector<srtb::real>& dms,
                               const std::string& who) {
  const size_t n = (size_t)std::min<uint64_t>(n_events, cap);
  if (n_events > cap)
    SRTB_LOGW << " [dm_search_candidates] " << who << ": " << n_events << " events, only the first " << cap
              << " clustered";
  std::vector<srtb_b200_candidate> c(std::max<size_t>(n, 1));
  uint64_t n_c = 0;
  if (srtb_b200_cluster_events(events, n, dms.data(), dms.size(), c.data(), c.size(), &n_c) != 0)
    throw std::runtime_error(std::string{"[dm_search_candidates] "} + srtb_b200_last_error(nullptr));
  for (size_t i = 0; i < std::min<uint64_t>(n_c, c.size()); i++)
    out.push_back({c[i].snr, c[i].dm, c[i].dm_low, c[i].dm_high, c[i].boxcar_length, c[i].peak_index, c[i].window,
                   c[i].members, c[i].span_begin, c[i].span_end, c[i].trial});
}

/** dm_search_candidates: stream s's events (at most cap of the true total n_events) clustered into w's candidates; a
 *  warning names both counts when the cap cut the list */
inline void attach_candidates(srtb::work::write_signal_work& w, const srtb_b200_event* events, uint64_t n_events,
                              size_t cap, const std::vector<srtb::real>& dms, uint64_t sample_offset) {
  cluster_candidates(w.candidates, events, n_events, cap, dms, "stream " + std::to_string(w.data_stream_id));
  w.has_candidates = true;
  w.candidate_share = candidate_share(w);
  w.candidate_sample_offset = sample_offset;
}

/** candidate_cutouts' fixed geometry: W = n_rows = 256, nsub = the largest divisor of C up to 256 */
constexpr size_t cutout_width = 256, cutout_rows = 256;
inline size_t cutout_nsub(size_t C) {
  for (size_t d = std::min<size_t>(C, 256); d > 1; d--)
    if (C % d == 0) return d;
  return 1;
}

/** max_c |k[c]|: the largest residual delay per unit DM over the band, in spectrum samples (k[c] as
 *  srtb_b200_candidate_cutouts defines it, the same expression and order) */
inline double cutout_k_max(size_t C, float freq_low, float bandwidth, float sample_rate) {
  const double f_ref = (double)(float)(freq_low + bandwidth);
  const double scale = (double)sample_rate / (2.0 * (double)C);
  double k_max = 0;
  for (size_t c = 0; c < C; c++) {
    const double f = (double)freq_low + (double)bandwidth * ((double)c + 0.5) / (double)C;
    k_max = std::max(k_max, std::fabs((1.0 / (f * f) - 1.0 / (f_ref * f_ref)) * scale * 4.148808e3));
  }
  return k_max;
}

/** the plane's DM half-width: (W/2) q / max_c |k[c]|, the DM offset whose residual sweep across the band fills half the
 *  image, so the bow tie of a pulse at the candidate's DM spans the plane (0 for a band without dispersion) */
inline float cutout_halfwidth(size_t W, uint32_t q, double k_max) {
  return k_max > 0 ? (float)((double)(W / 2) * (double)q / k_max) : 0.f;
}

/** the rows of a candidate file (those below share, in file order) to cut out: the n highest-S/N, highest first, ties
 *  in file order. Returns (row in the file, index into candidates) */
inline std::vector<std::pair<uint64_t, size_t>> cutout_selection(const std::vector<srtb::work::dm_candidate>& candidates,
                                                                 uint64_t share, size_t n) {
  std::vector<std::pair<uint64_t, size_t>> rows;
  for (size_t i = 0; i < candidates.size(); i++)
    if (candidates[i].window < share) rows.push_back({rows.size(), i});
  std::stable_sort(rows.begin(), rows.end(),
                   [&](const auto& a, const auto& b) { return candidates[a.second].snr > candidates[b.second].snr; });
  if (rows.size() > n) rows.resize(n);
  return rows;
}

/** the cut-out requests of a selection: q = max(1, boxcar_length / 2), center = window + offset + boxcar_length / 2,
 *  the candidate's DM, half-width by cutout_halfwidth */
inline std::vector<srtb_b200_cutout_request> cutout_requests(const std::vector<srtb::work::dm_candidate>& candidates,
                                                             const std::vector<std::pair<uint64_t, size_t>>& sel,
                                                             uint64_t sample_offset, double k_max) {
  std::vector<srtb_b200_cutout_request> out;
  for (const auto& [row, i] : sel) {
    const srtb::work::dm_candidate& c = candidates[i];
    srtb_b200_cutout_request r{};
    r.decimation = (uint32_t)std::max<uint64_t>(1, c.boxcar_length / 2);
    r.center = (int64_t)(c.window + sample_offset + c.boxcar_length / 2);
    r.dm = c.dm;
    r.dm_halfwidth = cutout_halfwidth(cutout_width, r.decimation, k_max);
    out.push_back(r);
  }
  return out;
}

/** events per stream and block a DM search lists for its candidates (dm_search_candidates) */
constexpr size_t candidate_event_cap = (size_t)1 << 18;

/** events per stream (and sum) and block the block path lists for its candidates (signal_detect_candidates): 2.5 MiB
 *  of pinned list per detector and ring slot. A row of L' samples holds at most L'/2 runs, so a config #3 block
 *  (L = 2^14, 9 boxcars) could exceed it only when most of its samples sit above threshold, i.e. on RFI; noise at the
 *  configured threshold lists a handful. Above the cap the first events in (boxcar, begin) order are clustered. */
constexpr size_t block_candidate_event_cap = (size_t)1 << 16;

class baseband_chain_pipe {
 protected:
  srtb::cuda_queue q;
  block_config_holder holder;
  struct pending_block {
    int ticket;
    int streams;
    size_t C, L;
    srtb::work::copy_to_device_work work;
    // what the block leaves behind, owned by the work items it turns into (zero copy, like the reference's d_in):
    std::vector<std::shared_ptr<srtb::complex<srtb::real>>> d_spectrum;  // per stream: N + 2 floats, [C][L] when done
    std::shared_ptr<srtb::real> h_series;  // pinned [streams (+ 1 with the sum)][MAX_BOXCARS][L]
    bool sum = false;                       // signal_detect_sum_streams: the sum's result follows the streams'
    bool events = false;                    // signal_detect_candidates: submitted through submit_block_events
    srtb::real dm = 0;                      // the block's dm, which its candidates carry
  };
  std::deque<pending_block> pending;  // blocks in the pinned-host ring of this queue's context
  std::vector<srtb_b200_event> events;  // dm_search_candidates: one stream's events, reused

 public:
  /** ring_depth blocks are kept in flight through srtb_b200_submit_block_ex / collect_block_ex (block k's H2D
   *  overlaps block k-1's compute; results lag the input by ring_depth - 1 works and an idle tick from
   *  idle_queue_in_functor flushes). ring_depth <= 1: every work is collected before operator() returns.
   *  Every write_signal_work carries its dynamic spectrum (work.ptr) and the host series of its positive boxcars,
   *  exactly what signal_detect_pipe_2 forwards (signal_detect_pipe.hpp:347-366,405-441): write_signal_pipe's
   *  "neighbour of a positive" rule (write_signal_pipe.hpp:102-115) therefore sees a spectrum on negatives too.
   *  keep_every_spectrum is kept for source compatibility; spectra are always kept now. */
  explicit baseband_chain_pipe(srtb::cuda_queue q_, bool keep_every_spectrum_ = false, int ring_depth_ = 1)
      : q{q_}, keep_every_spectrum{keep_every_spectrum_},
        ring_depth{std::max(1, std::min(ring_depth_, (int)SRTB_B200_RING_SLOTS))} {}

  using out_type = std::vector<srtb::work::write_signal_work>;

  std::optional<out_type> operator()(std::stop_token, srtb::work::copy_to_device_work in_work) {
    cuda_check(cudaSetDevice(q.device()), "cudaSetDevice");
    const bool idle_tick = (in_work.count == 0 && !in_work.baseband_data.baseband_ptr);
    out_type out;
    if (!idle_tick) submit(std::move(in_work));
    while (!pending.empty() && (idle_tick || (int)pending.size() >= ring_depth)) collect_front(out);
    return std::optional{std::move(out)};
  }

  bool keep_every_spectrum = false;
  int ring_depth = 1;

 protected:
  void submit(srtb::work::copy_to_device_work in_work) {
    holder.refresh();
    const auto& cfg = holder.cfg;
    pending_block p;
    p.streams = block_config_holder::stream_count(cfg.baseband_format);
    const size_t N = cfg.baseband_input_count, Nc = N / 2;
    p.C = std::min<size_t>(cfg.spectrum_channel_count, Nc);
    p.L = p.C ? Nc / p.C : 0;
    srtb_b200_block_outputs outputs{};
    for (int s = 0; s < p.streams; s++) {
      p.d_spectrum.push_back(srtb::device_allocator.allocate_shared<srtb::complex<srtb::real>>(Nc + 1));
      outputs.d_spectrum[s] = reinterpret_cast<float*>(p.d_spectrum.back().get());
    }
    p.sum = cfg.signal_detect_sum_streams != 0;
    p.h_series = srtb::host_allocator.allocate_shared<srtb::real>((size_t)(p.streams + (p.sum ? 1 : 0)) *
                                                                  SRTB_B200_MAX_BOXCARS * p.L);
    outputs.h_series = p.h_series.get();
    p.events = srtb::config.signal_detect_candidates;
    p.dm = cfg.dm;
    if (p.events)
      p.ticket = srtb_b200_submit_block_events(q.ctx(), &cfg, in_work.baseband_data.baseband_ptr.get(),
                                               in_work.baseband_data.baseband_input_bytes, /*on_device=*/0, &outputs,
                                               block_candidate_event_cap);
    else
      p.ticket = srtb_b200_submit_block_ex(q.ctx(), &cfg, in_work.baseband_data.baseband_ptr.get(),
                                           in_work.baseband_data.baseband_input_bytes, /*on_device=*/0, &outputs);
    q.check(p.ticket);
    p.work = std::move(in_work);
    pending.push_back(std::move(p));
  }

  void collect_front(out_type& out) {
    pending_block p = std::move(pending.front());
    pending.pop_front();
    srtb_b200_detect_result res[5];
    const srtb_b200_event* ev_list = nullptr;
    uint64_t n_ev[5] = {0, 0, 0, 0, 0};
    const int n = p.events ? srtb_b200_collect_block_events(q.ctx(), p.ticket, res, nullptr, nullptr, &ev_list, n_ev)
                           : srtb_b200_collect_block_ex(q.ctx(), p.ticket, res, nullptr, nullptr);
    q.check(n);
    // signal_detect_candidates: the slot's list is [streams (+1)][cap], clustered at the block's one DM
    const std::vector<srtb::real> block_dm{p.dm};
    constexpr size_t cap = block_candidate_event_cap;
    // fold_period: the block's fold, for the sink's accumulator (blocks not read from a file are not folded)
    std::shared_ptr<const srtb::work::fold_block> fold;
    if (srtb::config.fold_period != 0 && p.work.first_sample != p.work.no_first_sample) fold = fold_front(p);
    bool sum_positive = false;
    if (p.sum)
      for (int b = 0; b < res[n].n_boxcars; b++) sum_positive = sum_positive || res[n].signal_count[b] > 0;
    // incoherent_dm_list: the trial DMs searched around dm on each stream's dynamic spectrum
    const std::vector<srtb::real> inc_dms = srtb::program_options::parse_dm_list(srtb::config.incoherent_dm_list);
    std::shared_ptr<srtb::real> h_inc;
    if (!inc_dms.empty())
      h_inc = srtb::host_allocator.allocate_shared<srtb::real>((size_t)p.streams * SRTB_B200_MAX_BOXCARS * p.L);
    for (int s = 0; s < n; s++) {
      srtb::work::write_signal_work w;
      w.copy_parameter_from(p.work);
      w.data_stream_id = p.work.data_stream_id * static_cast<uint32_t>(p.streams) + static_cast<uint32_t>(s);
      w.count = p.L;
      w.batch_size = p.C;
      w.zero_count = res[s].zero_count;
      w.ptr = p.d_spectrum[s];
      w.sum_positive = sum_positive;
      if (s == 0) w.fold = fold;
      if (p.sum && s == 0) {
        w.carries_sum = true;
        w.sum_zero_count = res[n].zero_count;
        for (int b = 0; b < res[n].n_boxcars; b++) w.sum_signal_count.push_back(res[n].signal_count[b]);
        w.sum_time_series = positive_series(res[n], p.h_series, n, p.L);
      }
      if (p.events) {
        attach_candidates(w, ev_list + (size_t)s * cap, n_ev[s], cap, block_dm, 0);
        w.cutouts = cut_out(p, w, w.candidates, {s}, p.L - res[s].time_series_count);
        if (p.sum && s == 0) {
          cluster_candidates(w.sum_candidates, ev_list + (size_t)n * cap, n_ev[n], cap, block_dm, "sum");
          w.has_sum_candidates = true;
          std::vector<int> all(p.streams);
          for (int t = 0; t < p.streams; t++) all[t] = t;
          w.sum_cutouts = cut_out(p, w, w.sum_candidates, all, p.L - res[n].time_series_count);
        }
      }
      if (inc_dms.empty())
        w.time_series = positive_series(res[s], p.h_series, s, p.L);
      else
        incoherent_search(w, p, s, res[s], inc_dms, h_inc);
      out.push_back(std::move(w));
    }
  }

  /** candidate_cutouts: the cut-outs of the highest-S/N candidates of `candidates` (those below w's share) on the
   *  spectra of `streams` (stream indices into p.d_spectrum), or null when the key is off or none is listed */
  std::shared_ptr<const srtb::work::cutout_set> cut_out(const pending_block& p, const srtb::work::write_signal_work& w,
                                                        const std::vector<srtb::work::dm_candidate>& candidates,
                                                        const std::vector<int>& streams, size_t time_reserved_count) {
    const int64_t N = srtb::config.candidate_cutouts;
    if (N <= 0) return nullptr;
    const auto sel = cutout_selection(candidates, w.candidate_share, (size_t)N);
    if (sel.empty()) return nullptr;
    const auto& cfg = holder.cfg;
    const double k_max = cutout_k_max(p.C, cfg.baseband_freq_low, cfg.baseband_bandwidth, cfg.baseband_sample_rate);
    const auto req = cutout_requests(candidates, sel, w.candidate_sample_offset, k_max);
    auto out = std::make_shared<srtb::work::cutout_set>();
    out->width = cutout_width;
    out->nsub = cutout_nsub(p.C);
    out->n_rows = cutout_rows;
    out->ft.resize(req.size() * out->nsub * out->width);
    out->dmt.resize(req.size() * out->n_rows * out->width);
    std::vector<float> row_dms(req.size() * out->n_rows);
    std::vector<const void*> spectra;
    for (int s : streams) spectra.push_back(p.d_spectrum[s].get());
    q.check(srtb_b200_candidate_cutouts(q.ctx(), spectra.data(), (int)spectra.size(), p.L, p.C, time_reserved_count,
                                        cfg.baseband_freq_low, cfg.baseband_bandwidth, cfg.baseband_sample_rate,
                                        cfg.dm, req.data(), req.size(), out->width, out->nsub, out->n_rows,
                                        out->ft.data(), out->dmt.data(), row_dms.data()));
    for (size_t i = 0; i < req.size(); i++)
      out->rows.push_back({sel[i].first, req[i].center, req[i].decimation, row_dms[i * out->n_rows],
                           row_dms[i * out->n_rows + out->n_rows - 1]});
    return out;
  }

  /** folds the block's streams at fold_period: the first min(block step, samples read) / (2C) spectrum samples */
  std::shared_ptr<const srtb::work::fold_block> fold_front(const pending_block& p) {
    const auto& c = srtb::config;
    const uint64_t two_c = 2 * (uint64_t)p.C, step = fold_block_step();
    auto f = std::make_shared<srtb::work::fold_block>();
    f->block_index = p.work.first_sample / step;
    f->first_sample = p.work.first_sample;
    f->streams = (size_t)p.streams;
    f->subbands = c.fold_subband_count;
    f->bins = c.fold_bin_count;
    f->profile.assign(f->streams * f->subbands * f->bins, 0.0);
    f->hits.assign(f->bins, 0);
    f->kept.assign(f->streams * f->subbands, 0);
    const size_t fold_count = (size_t)std::min<uint64_t>(std::min(step, p.work.valid_samples) / two_c, p.L);
    if (c.fold_coherence) {
      f->coherence.assign(4 * f->subbands * f->bins, 0.0);
      f->coherence_kept.assign(f->subbands, 0);
    }
    if (fold_count == 0) return f;  // nothing read past the previous block's share: an empty fold keeps the order
    double phi0 = 0, a = 0, b = 0;
    q.check(srtb_b200_fold_phase(c.fold_period, c.fold_period_derivative, c.baseband_sample_rate, two_c,
                                 p.work.first_sample, &phi0, &a, &b));
    const void* spectra[4] = {};
    for (int s = 0; s < p.streams; s++) spectra[s] = p.d_spectrum[s].get();
    q.check(srtb_b200_fold(q.ctx(), spectra, p.streams, p.L, p.C, fold_count, phi0, a, b, f->bins, f->subbands,
                           f->profile.data(), f->hits.data(), f->kept.data()));
    if (c.fold_coherence)  // streams 0 and 1 are the two feeds (check_fold); the same samples, bins and hits
      q.check(srtb_b200_fold_coherence(q.ctx(), spectra[0], spectra[1], p.L, p.C, fold_count, phi0, a, b, f->bins,
                                       f->subbands, f->coherence.data(), f->hits.data(), f->coherence_kept.data()));
    return f;
  }

  /** the incoherent search of stream s's spectrum: fills w's DM-search fields as dm_sweep_chain_pipe does (best trial's
   *  DM and positive series, one summary per trial), so write_signal_pipe writes its .dm<DM>.<boxcar>.tim files and
   *  dm_sweep.csv; the work is positive when the best trial is */
  void incoherent_search(srtb::work::write_signal_work& w, const pending_block& p, int s,
                         const srtb_b200_detect_result& block_res, const std::vector<srtb::real>& dms,
                         const std::shared_ptr<srtb::real>& h_inc) {
    const auto& cfg = holder.cfg;
    const size_t n_dm = dms.size();
    std::vector<srtb_b200_detect_result> tr(n_dm);
    std::vector<srtb_b200_peak> peaks(n_dm);
    int32_t best = 0;
    if (srtb::config.dm_search_candidates) {
      events.resize(candidate_event_cap);
      uint64_t n_events = 0, s_minus = 0;
      q.check(srtb_b200_incoherent_dm_search_events(
          q.ctx(), p.d_spectrum[s].get(), p.L, p.C, p.L - block_res.time_series_count, cfg.baseband_freq_low,
          cfg.baseband_bandwidth, cfg.baseband_sample_rate, cfg.dm, dms.data(), n_dm,
          cfg.signal_detect_signal_noise_threshold, cfg.signal_detect_channel_threshold,
          cfg.signal_detect_max_boxcar_length, tr.data(), peaks.data(), &best,
          h_inc.get() + (size_t)s * SRTB_B200_MAX_BOXCARS * p.L, events.data(), events.size(), &n_events));
      q.check(srtb_b200_incoherent_shifts(p.C, cfg.baseband_freq_low, cfg.baseband_bandwidth, cfg.baseband_sample_rate,
                                          cfg.dm, dms.data(), n_dm, nullptr, nullptr, &s_minus));
      attach_candidates(w, events.data(), n_events, events.size(), dms, s_minus);
      w.cutouts = cut_out(p, w, w.candidates, {s}, p.L - block_res.time_series_count);
    } else {
      q.check(srtb_b200_incoherent_dm_search(
          q.ctx(), p.d_spectrum[s].get(), p.L, p.C, p.L - block_res.time_series_count, cfg.baseband_freq_low,
          cfg.baseband_bandwidth, cfg.baseband_sample_rate, cfg.dm, dms.data(), n_dm,
          cfg.signal_detect_signal_noise_threshold, cfg.signal_detect_channel_threshold,
          cfg.signal_detect_max_boxcar_length, tr.data(), peaks.data(), &best,
          h_inc.get() + (size_t)s * SRTB_B200_MAX_BOXCARS * p.L));
    }
    const srtb_b200_detect_result& r = tr[best];
    w.time_series = positive_series(r, h_inc, s, p.L, r.time_series_count);
    w.dm = dms[best];
    w.dm_trials = dm_trials(tr.data(), peaks.data(), dms, 1, 0);
  }
};

}  // namespace pipeline
}  // namespace srtb
