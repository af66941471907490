// srtb/config.hpp — the srtb::configs surface the hot path reads, field for field
// (reference: userspace/include/srtb/config.hpp:28-58 compile-time knobs, :80-249 struct configs).
// GUI / FFTW-only fields are kept so the shipped .cfg files still map onto the struct.
#pragma once
#include <complex>
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

namespace srtb {

using real = float;                       // math.hpp:44
template <typename T>
using complex = std::complex<T>;          // layout-compatible with float2 on the device

inline constexpr size_t work_queue_capacity = 2;      // config.hpp:40
inline constexpr bool work_queue_fixed_size = true;   // config.hpp:43
inline constexpr bool fft_window_precompute = false;  // config.hpp:46
inline constexpr bool fft_operate_in_place = true;    // config.hpp:47
inline constexpr size_t MEMORY_ALIGNMENT = 64ul;      // config.hpp:56
inline constexpr size_t BITS_PER_BYTE = 8ul;          // config.hpp:58

// waterfall thumbnail colours, ARGB32 (config.hpp:60-68): intensity 0 -> color_0, 1 -> color_1, else color_overflow
namespace gui {
inline constexpr uint32_t opaque = 0xff000000;
inline constexpr uint32_t color_0 = 0x1f1e33 | opaque;
inline constexpr uint32_t color_1 = 0x33e1f1 | opaque;
inline constexpr uint32_t color_overflow = 0xe0e1cc | opaque;
}  // namespace gui

struct configs {
  std::string config_file_name = "srtb_config.cfg";
  size_t baseband_input_count = size_t{1} << 28;
  int32_t baseband_input_bits = 8;
  std::string baseband_format_type = "simple";
  srtb::real baseband_freq_low = 1000.0;
  srtb::real baseband_bandwidth = 500.0;
  srtb::real baseband_sample_rate = 1000 * 1e6;
  bool baseband_reserve_sample = true;
  srtb::real dm = 0;
  // trial DMs searched on every block instead of `dm` (new with respect to the reference, whose config.hpp:128-132
  // leaves a DM search list as a TODO): comma-separated expressions or start:stop:step ranges; empty = search `dm` only
  std::string dm_list = "";
  // trial DMs searched incoherently around `dm` on every block's dynamic spectrum (semi-coherent search: coherent at
  // `dm`, then each trial's residual delay between channels as a whole-sample shift); same syntax as dm_list, and
  // not together with it. Empty = no incoherent search
  std::string incoherent_dm_list = "";
  // also run the single-pulse detector on the total intensity of a block's streams (polarisations), sum_s |x_s|^2 over
  // the channels no stream masks: sqrt(2) the S/N of either polarisation for an unpolarised pulse. Needs a format of
  // two or more streams; not with dm_list or incoherent_dm_list
  bool signal_detect_sum_polarizations = false;
  // fold every block of a recording at a known pulsar period (seconds; 0 = off) with derivative fold_period_derivative
  // (s/s) into fold_bin_count phase bins and fold_subband_count subbands of consecutive channels; subintegrations of
  // fold_subintegration_blocks blocks (0 = one for the whole run). Phase and time reference: include/srtb_b200.h
  double fold_period = 0;
  double fold_period_derivative = 0;
  size_t fold_bin_count = 256;
  size_t fold_subband_count = 1;
  size_t fold_subintegration_blocks = 0;
  // with fold_period: also fold the coherence products AA, BB, CR, CI of streams 0 and 1 (the two feeds of a
  // dual-polarisation format) over the channels kept in both; needs a two-stream format (not gznupsr_a1_4)
  bool fold_coherence = false;
  // with dm_list or incoherent_dm_list: also list each block's single-pulse candidates, every above-threshold run of
  // every trial and boxcar grouped friends-of-friends over DM, width and time (<prefix><counter>.<id>.candidates.csv)
  bool dm_search_candidates = false;
  // the block path (no DM search): also list each block's single-pulse candidates at its one dm, every above-threshold
  // run of every stream's boxcar series grouped friends-of-friends over width and time (<prefix><counter>.<id>.candidates
  // .csv), and the total intensity's with signal_detect_sum_polarizations (<prefix><counter>.sum.candidates.csv)
  bool signal_detect_candidates = false;
  // with signal_detect_candidates or dm_search_candidates: cut out the N highest-S/N candidates of each candidate file
  // (0 = off): the dedispersed frequency-time image and the DM-time plane of each (<prefix><counter>.<id>.cutout_ft.npy,
  // .cutout_dmt.npy, .cutouts.csv), from the block's spectra on the device; not with dm_list
  int64_t candidate_cutouts = 0;
  std::vector<std::string> udp_receiver_address = {"10.0.1.2"};
  std::vector<unsigned short> udp_receiver_port = {12004};
  std::vector<uint32_t> udp_receiver_cpu_preferred = {0};
  std::string input_file_path = "";
  size_t input_file_offset_bytes = 0;
  std::string baseband_output_file_prefix = "srtb_baseband_output_";
  bool baseband_write_all = false;
  std::string fft_fftw_wisdom_path = "srtb_fftw_wisdom.txt";
  srtb::real mitigate_rfi_average_method_threshold = 10;
  srtb::real mitigate_rfi_spectral_kurtosis_threshold = 1.1;
  std::string mitigate_rfi_freq_list = "";
  size_t spectrum_sum_count = 1;
  size_t spectrum_channel_count = size_t{1} << 15;
  srtb::real signal_detect_signal_noise_threshold = 6;
  srtb::real signal_detect_channel_threshold = 0.9;
  size_t signal_detect_max_boxcar_length = 1024;
  size_t thread_query_work_wait_time = 1000;
  bool gui_enable = false;
  size_t gui_pixmap_width = 1920;
  size_t gui_pixmap_height = 1080;
};

// the one global every pipe re-reads at call time (global_variables.hpp:42)
inline srtb::configs config;

}  // namespace srtb
