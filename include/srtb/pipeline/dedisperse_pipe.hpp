// srtb/pipeline/dedisperse_pipe.hpp — coherent dedispersion pipe
// (reference: userspace/include/srtb/pipeline/dedisperse_pipe.hpp:27-48): df = bandwidth / N,
// f_min = freq_low, f_c = freq_low + bandwidth, all float (SURVEY q7), read from config per call.
#pragma once
#include <algorithm>
#include <optional>
#include <stdexcept>
#include <stop_token>
#include <string>
#include <vector>

#include "srtb/config.hpp"
#include "srtb/cuda_queue.hpp"
#include "srtb/pipeline/mode.hpp"
#include "srtb/program_options.hpp"  // parse_dm_list
#include "srtb/work.hpp"

namespace srtb {
namespace coherent_dedispersion {
/** reference: coherent_dedispersion.hpp:103-128 (reads the global config; may clear reserve_sample) */
inline size_t nsamps_reserved() {
  const size_t r = srtb_b200_nsamps_reserved(
      srtb::config.baseband_input_count, srtb::config.spectrum_channel_count, srtb::config.baseband_freq_low,
      srtb::config.baseband_bandwidth, srtb::config.baseband_sample_rate, srtb::config.dm,
      srtb::config.baseband_reserve_sample ? 1 : 0);
  if (r == 0 && srtb::config.baseband_reserve_sample) srtb::config.baseband_reserve_sample = false;
  return r;
}

/** the block overlap the file reader rewinds and the baseband writer trims. With incoherent_dm_list (and
 *  baseband_reserve_sample): nsamps_reserved() + 2C (S+ + S-). Otherwise nsamps_reserved() without a dm_list, else
 *  the largest srtb_b200_nsamps_reserved over the trial DMs, so the trial with the largest dispersive smear still sees
 *  every pulse whole. The maximum is taken of the function itself: the sign of the delay depends on the signs of the DM
 *  and the bandwidth. Each trial's detector still leaves out only its own reserved tail, so trials with a smaller smear
 *  search part of the overlap in both blocks. */
/** S+ + S-: the samples of the dynamic spectrum the incoherent search (incoherent_dm_list) shifts its trials over, the
 *  C of the block path (spectrum_channel_count, at most N / 2); 0 without a list */
inline uint64_t incoherent_span() {
  const auto& c = srtb::config;
  const std::vector<srtb::real> dms = srtb::program_options::parse_dm_list(c.incoherent_dm_list);
  if (dms.empty()) return 0;
  const size_t C = std::min<size_t>(c.spectrum_channel_count, c.baseband_input_count / 2);
  uint64_t s_plus = 0, s_minus = 0;
  if (srtb_b200_incoherent_shifts(C, c.baseband_freq_low, c.baseband_bandwidth, c.baseband_sample_rate, c.dm,
                                  dms.data(), dms.size(), nullptr, &s_plus, &s_minus) != 0)
    throw std::invalid_argument("[dedisperse] incoherent_dm_list: " + std::string{srtb_b200_last_error(nullptr)});
  return s_plus + s_minus;
}

inline size_t nsamps_reserved_max() {
  if (!srtb::config.incoherent_dm_list.empty()) {
    // the incoherent search's trials read S+ + S- spectrum samples (2C baseband samples each) past the series it
    // searches: the next block repeats them, so a pulse there is searched whole in one of the two blocks
    if (!srtb::config.baseband_reserve_sample) return nsamps_reserved();
    const size_t C = std::min<size_t>(srtb::config.spectrum_channel_count, srtb::config.baseband_input_count / 2);
    return nsamps_reserved() + 2 * C * (size_t)incoherent_span();
  }
  if (srtb::config.dm_list.empty()) return nsamps_reserved();
  const auto& c = srtb::config;
  size_t r = 0;
  for (const srtb::real dm : srtb::program_options::parse_dm_list(c.dm_list))
    r = std::max(r, srtb_b200_nsamps_reserved(c.baseband_input_count, c.spectrum_channel_count, c.baseband_freq_low,
                                              c.baseband_bandwidth, c.baseband_sample_rate, dm,
                                              c.baseband_reserve_sample ? 1 : 0));
  return r;
}
}  // namespace coherent_dedispersion
namespace codd = coherent_dedispersion;

namespace pipeline {

class dedisperse_pipe {
 public:
  srtb::cuda_queue q;
  explicit dedisperse_pipe(srtb::cuda_queue q_) : q{q_} {}

  auto operator()(std::stop_token, srtb::work::dedisperse_work in_work) {
    const size_t N = in_work.count;
    const srtb::real df = srtb::config.baseband_bandwidth / N;
    const srtb::real f_min = srtb::config.baseband_freq_low, f_c = f_min + srtb::config.baseband_bandwidth;
    const srtb::real dm = srtb::config.dm;
    cuda_check(cudaSetDevice(q.device()), "cudaSetDevice");
    q.check(srtb_b200_dedisperse(q.ctx(), in_work.ptr.get(), N, f_min, f_c, df, dm));
    end_of_pipe(q);
    srtb::work::watfft_1d_c2c_work out;
    auto ptr = in_work.ptr;
    out.move_parameter_from(std::move(in_work));
    out.ptr = ptr;
    out.count = N;
    out.batch_size = 1;
    return std::optional{out};
  }
};

}  // namespace pipeline
}  // namespace srtb
