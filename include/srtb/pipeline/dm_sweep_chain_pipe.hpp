// srtb/pipeline/dm_sweep_chain_pipe.hpp — the device chain as one pipe, searching a list of trial DMs (config
// dm_list) instead of the one `dm`. Same input and output as baseband_chain_pipe, so main.cpp wires it the same way:
// it takes the copy_to_device_work a source pipe produced and returns one write_signal_work per data stream.
// Each block is one synchronous srtb_b200_process_block_dm_sweep_ex call: unpack and R2C once per stream, then s1,
// chirp, waterfall FFT, SK and the detector for every trial, and the stream's best trial once more to hand out its
// dynamic spectrum and positive series. Blocks overlap on the GPU across the several pipes (one context each) that
// pop from one work queue; there is no ring inside the pipe.
#pragma once
#include <memory>
#include <optional>
#include <stdexcept>
#include <stop_token>
#include <vector>

#include "srtb/config.hpp"
#include "srtb/cuda_queue.hpp"
#include "srtb/memory.hpp"
#include "srtb/pipeline/baseband_chain_pipe.hpp"  // block_config_holder, positive_series
#include "srtb/program_options.hpp"               // parse_dm_list
#include "srtb/work.hpp"

namespace srtb {
namespace pipeline {

class dm_sweep_chain_pipe {
 protected:
  srtb::cuda_queue q;
  block_config_holder holder;
  std::vector<srtb_b200_event> events;  // dm_search_candidates: [streams][candidate_event_cap], reused

 public:
  explicit dm_sweep_chain_pipe(srtb::cuda_queue q_) : q{q_} {}

  using out_type = std::vector<srtb::work::write_signal_work>;

  /** Every write_signal_work carries the best trial's dynamic spectrum (work.ptr) and positive series (time_series,
   *  non-empty exactly when some trial is positive), its DM (dm) and one summary per trial (dm_trials). */
  std::optional<out_type> operator()(std::stop_token, srtb::work::copy_to_device_work in_work) {
    out_type out;
    if (in_work.count == 0 && !in_work.baseband_data.baseband_ptr) return std::optional{std::move(out)};  // idle tick
    cuda_check(cudaSetDevice(q.device()), "cudaSetDevice");
    holder.refresh();
    const std::vector<srtb::real> dms = srtb::program_options::parse_dm_list(srtb::config.dm_list);
    if (dms.empty()) throw std::invalid_argument("[dm_sweep_chain_pipe] dm_list is empty");
    const auto& cfg = holder.cfg;
    const int streams = block_config_holder::stream_count(cfg.baseband_format);
    const size_t N = cfg.baseband_input_count, Nc = N / 2;
    const size_t C = std::min<size_t>(cfg.spectrum_channel_count, Nc), L = C ? Nc / C : 0;
    const size_t n_dm = dms.size();

    std::vector<std::shared_ptr<srtb::complex<srtb::real>>> d_spectrum;
    srtb_b200_sweep_outputs outputs{};
    for (int s = 0; s < streams; s++) {
      d_spectrum.push_back(srtb::device_allocator.allocate_shared<srtb::complex<srtb::real>>(Nc + 1));
      outputs.d_spectrum[s] = reinterpret_cast<float*>(d_spectrum.back().get());
    }
    auto h_series = srtb::host_allocator.allocate_shared<srtb::real>((size_t)streams * SRTB_B200_MAX_BOXCARS * L);
    outputs.h_series = h_series.get();
    std::vector<srtb_b200_detect_result> res(n_dm * streams);
    std::vector<srtb_b200_peak> peaks(n_dm * streams);
    int32_t best[4] = {0, 0, 0, 0};
    outputs.h_peaks = peaks.data();
    outputs.h_best_trial = best;
    const bool candidates = srtb::config.dm_search_candidates;
    uint64_t n_events[4] = {0, 0, 0, 0};
    if (candidates) {
      events.resize((size_t)streams * candidate_event_cap);
      q.check(srtb_b200_process_block_dm_sweep_events(
          q.ctx(), &cfg, in_work.baseband_data.baseband_ptr.get(), in_work.baseband_data.baseband_input_bytes,
          /*on_device=*/0, dms.data(), n_dm, res.data(), &outputs, events.data(), candidate_event_cap, n_events));
    } else {
      q.check(srtb_b200_process_block_dm_sweep_ex(q.ctx(), &cfg, in_work.baseband_data.baseband_ptr.get(),
                                                  in_work.baseband_data.baseband_input_bytes, /*on_device=*/0,
                                                  dms.data(), n_dm, res.data(), &outputs));
    }

    for (int s = 0; s < streams; s++) {
      const srtb_b200_detect_result& r = res[(size_t)best[s] * streams + s];
      srtb::work::write_signal_work w;
      w.copy_parameter_from(in_work);
      w.data_stream_id = in_work.data_stream_id * static_cast<uint32_t>(streams) + static_cast<uint32_t>(s);
      w.count = L;
      w.batch_size = C;
      w.zero_count = r.zero_count;
      w.ptr = d_spectrum[s];
      w.time_series = positive_series(r, h_series, s, L);
      w.dm = dms[best[s]];
      w.dm_trials = dm_trials(res.data(), peaks.data(), dms, (size_t)streams, s);
      if (candidates)
        attach_candidates(w, events.data() + (size_t)s * candidate_event_cap, n_events[s], candidate_event_cap, dms, 0);
      out.push_back(std::move(w));
    }
    return std::optional{std::move(out)};
  }
};

}  // namespace pipeline
}  // namespace srtb
