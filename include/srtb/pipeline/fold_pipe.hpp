// srtb/pipeline/fold_pipe.hpp — the sink side of folding (fold_period): adds the per-block folds that
// baseband_chain_pipe attaches to each block's first work into subintegrations and writes them.
//
// Blocks reach the sink in any order when several chains or GPUs run; the accumulator holds early ones back and adds
// every block in block-index order, in float64, so the files do not depend on that order. Files, each written to a
// temporary name and renamed when a subintegration completes and at finish():
//   <baseband_output_file_prefix>fold.npy          float64 [subint][stream][subband][bin], the summed |x|^2
//   <baseband_output_file_prefix>fold.weights.npy  float64, the same shape: sum over blocks of kept[s][k] hits[bin], so
//                                                  fold / weights is the mean power per channel-sample
//   <baseband_output_file_prefix>fold.json         the parameters, each subintegration's start time and the reference;
//                                                  no wall-clock time, so two runs over one recording write the same bytes
// and with fold_coherence also
//   <baseband_output_file_prefix>fold.coherence.npy          float64 [subint][4][subband][bin]: AA, BB, CR, CI of
//                                                            X = stream 0 and Y = stream 1 (srtb_b200_fold_coherence)
//   <baseband_output_file_prefix>fold.coherence.weights.npy  float64 [subint][subband][bin]: sum over blocks of
//                                                            kept[k] hits[bin], kept counting the channels kept in both
#pragma once
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <filesystem>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "srtb/config.hpp"
#include "srtb/io/npy.hpp"
#include "srtb/log.hpp"
#include "srtb/pipeline/dedisperse_pipe.hpp"  // srtb::codd::nsamps_reserved_max
#include "srtb/work.hpp"

namespace srtb {
namespace pipeline {

/** baseband samples per stream from one block's start to the next's: N - R, R the overlap read_file_pipe rewinds
 *  (nsamps_reserved_max(), a multiple of 2C), or N when it does not rewind (R >= N). A block folds its first
 *  block_step / (2C) spectrum samples, so consecutive blocks fold every sample once */
inline uint64_t fold_block_step() {
  const size_t N = srtb::config.baseband_input_count, R = srtb::codd::nsamps_reserved_max();
  return R < N ? N - R : N;
}

/** the fold's fixed parameters, from srtb::config at start-up */
struct fold_parameters {
  double period = 0, period_derivative = 0, dm = 0, sample_rate = 0, freq_low = 0, bandwidth = 0;
  size_t streams = 1, channels = 0, subbands = 1, bins = 1;
  uint64_t block_step = 0;           // N - R: baseband samples per stream between consecutive blocks
  size_t subintegration_blocks = 0;  // 0 = one subintegration for the whole run
  bool coherence = false;            // fold_coherence: also the coherence products of streams 0 and 1
  std::string prefix;

  static fold_parameters from_config(size_t streams, uint64_t block_step) {
    const auto& c = srtb::config;
    fold_parameters p;
    p.period = c.fold_period;
    p.period_derivative = c.fold_period_derivative;
    p.dm = c.dm;
    p.sample_rate = c.baseband_sample_rate;
    p.freq_low = c.baseband_freq_low;
    p.bandwidth = c.baseband_bandwidth;
    p.streams = streams;
    p.channels = std::min<size_t>(c.spectrum_channel_count, c.baseband_input_count / 2);
    p.subbands = c.fold_subband_count;
    p.bins = c.fold_bin_count;
    p.block_step = block_step;
    p.subintegration_blocks = c.fold_subintegration_blocks;
    p.coherence = c.fold_coherence;
    p.prefix = c.baseband_output_file_prefix;
    return p;
  }
  double dt() const { return 2.0 * (double)channels / sample_rate; }
};

class fold_accumulator {
 public:
  explicit fold_accumulator(fold_parameters p) : par{std::move(p)} {}

  /** takes one block's fold; thread-safe. Blocks are added in block-index order once every earlier block is in */
  void add(std::shared_ptr<const srtb::work::fold_block> b) {
    std::lock_guard<std::mutex> g{m};
    if (b->streams != par.streams || b->subbands != par.subbands || b->bins != par.bins)
      throw std::runtime_error("[fold] a block's fold shape does not match the run's");
    if (par.coherence && (b->coherence.size() != 4 * par.subbands * par.bins ||
                          b->coherence_kept.size() != par.subbands))
      throw std::runtime_error("[fold] a block carries no coherence products of the run's shape");
    waiting[b->block_index] = std::move(b);
    bool completed = false;
    while (!waiting.empty() && waiting.begin()->first == next_block) {
      completed = fold_in(*waiting.begin()->second) || completed;
      waiting.erase(waiting.begin());
      next_block++;
    }
    if (completed) write();
  }

  /** adds what is still held back (in block-index order, past any block that never came) and writes the files */
  void finish() {
    std::lock_guard<std::mutex> g{m};
    for (auto& [index, b] : waiting) fold_in(*b);
    waiting.clear();
    if (blocks_folded) write();
  }

  uint64_t blocks() const {
    std::lock_guard<std::mutex> g{m};
    return blocks_folded;
  }
  size_t subintegrations() const {
    std::lock_guard<std::mutex> g{m};
    return subint_first.size();
  }

 private:
  fold_parameters par;
  mutable std::mutex m;
  std::map<uint64_t, std::shared_ptr<const srtb::work::fold_block>> waiting;
  uint64_t next_block = 0;
  uint64_t blocks_folded = 0;
  std::vector<double> profile, weights;  // [subint][stream][subband][bin]
  std::vector<double> coherence;         // [subint][4][subband][bin] (fold_coherence)
  std::vector<double> coherence_weights;  // [subint][subband][bin] (fold_coherence)
  std::vector<uint64_t> subint_first;    // first_sample of each subintegration's first block
  std::vector<uint64_t> subint_blocks;   // blocks added to each subintegration

  size_t row() const { return par.streams * par.subbands * par.bins; }

  // adds b; true when it is the last block of its subintegration
  bool fold_in(const srtb::work::fold_block& b) {
    const size_t si = par.subintegration_blocks ? (size_t)(b.block_index / par.subintegration_blocks) : 0;
    if (si >= subint_first.size()) {
      subint_first.resize(si + 1, 0);
      subint_blocks.resize(si + 1, 0);
      profile.resize((si + 1) * row(), 0.0);
      weights.resize((si + 1) * row(), 0.0);
      if (par.coherence) {
        coherence.resize((si + 1) * 4 * par.subbands * par.bins, 0.0);
        coherence_weights.resize((si + 1) * par.subbands * par.bins, 0.0);
      }
    }
    if (subint_blocks[si] == 0) subint_first[si] = b.first_sample;  // blocks come in index order
    subint_blocks[si]++;
    double* p = profile.data() + si * row();
    double* w = weights.data() + si * row();
    for (size_t sk = 0; sk < par.streams * par.subbands; sk++)
      for (size_t bin = 0; bin < par.bins; bin++) {
        p[sk * par.bins + bin] += b.profile[sk * par.bins + bin];
        w[sk * par.bins + bin] += (double)b.kept[sk] * (double)b.hits[bin];
      }
    if (par.coherence) {
      const size_t kb = par.subbands * par.bins;
      double* cp = coherence.data() + si * 4 * kb;
      double* cw = coherence_weights.data() + si * kb;
      for (size_t i = 0; i < 4 * kb; i++) cp[i] += b.coherence[i];
      for (size_t k = 0; k < par.subbands; k++)
        for (size_t bin = 0; bin < par.bins; bin++)
          cw[k * par.bins + bin] += (double)b.coherence_kept[k] * (double)b.hits[bin];
    }
    blocks_folded++;
    return par.subintegration_blocks && (b.block_index + 1) % par.subintegration_blocks == 0;
  }

  static std::string num(double v) {
    char buf[64];
    std::snprintf(buf, sizeof buf, "%.17g", v);
    return buf;
  }

  void write() const {
    const std::vector<size_t> shape = {subint_first.size(), par.streams, par.subbands, par.bins};
    const std::string base = par.prefix + "fold";
    const auto replace = [](const std::string& path, auto&& write_to) {
      const std::string tmp = path + ".tmp";
      write_to(tmp);
      std::filesystem::rename(tmp, path);
    };
    replace(base + ".npy", [&](const std::string& f) { srtb::io::npy_save(f, profile.data(), shape); });
    replace(base + ".weights.npy", [&](const std::string& f) { srtb::io::npy_save(f, weights.data(), shape); });
    if (par.coherence) {
      const size_t n = subint_first.size();
      const std::vector<size_t> cshape = {n, 4, par.subbands, par.bins}, wshape = {n, par.subbands, par.bins};
      replace(base + ".coherence.npy",
              [&](const std::string& f) { srtb::io::npy_save(f, coherence.data(), cshape); });
      replace(base + ".coherence.weights.npy",
              [&](const std::string& f) { srtb::io::npy_save(f, coherence_weights.data(), wshape); });
    }
    std::string starts, counts;
    for (size_t i = 0; i < subint_first.size(); i++) {
      starts += (i ? ", " : "") + num((double)subint_first[i] / par.sample_rate);
      counts += (i ? ", " : "") + std::to_string(subint_blocks[i]);
    }
    const std::string json =
        "{\n"
        "  \"period_s\": " + num(par.period) + ",\n"
        "  \"period_derivative\": " + num(par.period_derivative) + ",\n"
        "  \"dm\": " + num(par.dm) + ",\n"
        "  \"sample_rate_hz\": " + num(par.sample_rate) + ",\n"
        "  \"freq_low_mhz\": " + num(par.freq_low) + ",\n"
        "  \"bandwidth_mhz\": " + num(par.bandwidth) + ",\n"
        "  \"channels\": " + std::to_string(par.channels) + ",\n"
        "  \"streams\": " + std::to_string(par.streams) + ",\n"
        "  \"subbands\": " + std::to_string(par.subbands) + ",\n"
        "  \"bins\": " + std::to_string(par.bins) + ",\n"
        "  \"dt_s\": " + num(par.dt()) + ",\n"
        "  \"samples_per_block_step\": " + std::to_string(par.block_step) + ",\n"
        "  \"blocks_per_subintegration\": " + std::to_string(par.subintegration_blocks) + ",\n"
        "  \"blocks_folded\": " + std::to_string(blocks_folded) + ",\n"
        "  \"subintegration_blocks_folded\": [" + counts + "],\n"
        "  \"subintegration_start_s\": [" + starts + "],\n" +
        (par.coherence ? "  \"coherence\": [\"AA\", \"BB\", \"CR\", \"CI\"],\n"
                         "  \"coherence_definition\": \"X = stream 0, Y = stream 1; AA = |X|^2, BB = |Y|^2, "
                         "CR = Re(X conj Y), CI = Im(X conj Y), summed over the channels kept in both streams; "
                         "no calibration is applied\",\n"
                       : "") +
        "  \"reference\": \"t = 0 at the first sample after input_file_offset_bytes; topocentric, not barycentred; "
        "arrival times referred to freq_low + bandwidth, the frequency coherent dedispersion aligns the channels to; "
        "phase = t/P - (Pdot/P^2) t^2 / 2 with no timing-model predictor; bin 0 starts at phase 0\"\n"
        "}\n";
    replace(base + ".json", [&](const std::string& f) {
      std::FILE* fp = std::fopen(f.c_str(), "wb");
      if (!fp) throw std::runtime_error("[fold] cannot open " + f);
      std::fwrite(json.data(), 1, json.size(), fp);
      std::fclose(fp);
    });
  }
};

}  // namespace pipeline
}  // namespace srtb
