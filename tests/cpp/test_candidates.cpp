// CPU-only tests of the DM search candidates' host pieces: the dm_search_candidates key (include/srtb/program_options.hpp),
// the block's own share of candidate windows (candidate_share, include/srtb/pipeline/baseband_chain_pipe.hpp) and the
// <stem>.<id>.candidates.csv write_signal_pipe writes for a hand-made work: the share filter, the empty
// time of a block without a first sample, the header-only file. Links libsrtb_b200.so for its host arithmetic and
// needs no GPU.
#include <cstdio>
#include <filesystem>
#include <fstream>
#include <sstream>
#include <string>

#include "srtb/pipeline/baseband_chain_pipe.hpp"  // candidate_share
#include "srtb/pipeline/write_signal_pipe.hpp"
#include "srtb/program_options.hpp"

#define CHECK(...)                                                                             \
  do {                                                                                         \
    if (!(__VA_ARGS__)) {                                                                      \
      std::fprintf(stderr, "CHECK failed: %s (%s:%d)\n", #__VA_ARGS__, __FILE__, __LINE__); \
      return 1;                                                                                \
    }                                                                                          \
  } while (0)

static std::string read_text(const std::string& path) {
  std::ifstream f(path);
  std::stringstream ss;
  ss << f.rdbuf();
  return ss.str();
}

static srtb::work::dm_candidate cand(float snr, float dm, uint64_t boxcar, uint64_t window, uint64_t members) {
  srtb::work::dm_candidate c;
  c.snr = snr;
  c.dm = dm;
  c.dm_low = dm - 0.5f;
  c.dm_high = dm + 0.25f;
  c.boxcar_length = boxcar;
  c.window = window;
  c.peak_index = window - (boxcar > 1 ? 1 : 0);
  c.members = members;
  c.span_begin = window - 1;
  c.span_end = window + boxcar + 2;
  c.trial = 3;
  return c;
}

int main(int argc, char** argv) {
  srtb::log::current_level = srtb::log::levels::WARNING;
  const std::string dir = (argc > 1) ? argv[1] : "/tmp";
  using srtb::program_options::apply_changed_configs;
  using srtb::program_options::check_dm_search_candidates;

  // ---- the key, in a .cfg and on the command line, and the start-up check
  {
    srtb::configs c;
    CHECK(!c.dm_search_candidates);
    apply_changed_configs(srtb::program_options::parse_config_text("dm_search_candidates = 1\n"), c);
    CHECK(c.dm_search_candidates);
    apply_changed_configs({{"dm_search_candidates", "0"}}, c);
    CHECK(!c.dm_search_candidates);
    apply_changed_configs({{"dm_search_candidates", "1"}}, c);
    CHECK(c.dm_search_candidates);
    bool named = false;
    try {
      check_dm_search_candidates(c);
    } catch (const std::invalid_argument& e) {
      const std::string m = e.what();
      named = m.find("dm_search_candidates") != std::string::npos && m.find("dm_list") != std::string::npos &&
              m.find("incoherent_dm_list") != std::string::npos;
    }
    CHECK(named);
    c.dm_list = "1, 2";
    check_dm_search_candidates(c);
    c.dm_list = "";
    c.incoherent_dm_list = "3";
    check_dm_search_candidates(c);
    c.dm_search_candidates = false;
    c.incoherent_dm_list = "";
    check_dm_search_candidates(c);  // off: nothing to check
  }

  // ---- the sink. N = 65536, C = 16 (2C = 32), dm = 0: no overlap, step = N
  srtb::config.baseband_input_count = 65536;
  srtb::config.spectrum_channel_count = 16;
  srtb::config.baseband_sample_rate = 1e6;
  srtb::config.dm = 0;
  srtb::config.dm_list = "";
  srtb::config.incoherent_dm_list = "";
  CHECK(srtb::pipeline::fold_block_step() == 65536);
  using srtb::pipeline::write_signal_pipe;
  srtb::work::write_signal_work w;
  w.count = 2048;
  w.batch_size = 16;
  w.data_stream_id = 1;
  srtb::work::dm_trial_summary t;
  t.dm = 2;
  w.dm_trials.push_back(t);
  const std::string header = "snr,dm,boxcar_length,sample,time,members,dm_low,dm_high,span_begin,span_end,trial,"
                             "peak_index\n";
  // without the key's fields nothing is written
  write_signal_pipe::write_series(w, dir + "/none");
  CHECK(!std::filesystem::exists(dir + "/none.1.candidates.csv"));
  CHECK(std::filesystem::exists(dir + "/none.1.dm_sweep.csv"));

  // a block read from a file: the share is min(step, valid_samples) / 2C = 32000 / 32 = 1000
  w.has_candidates = true;
  w.first_sample = 320000;
  w.valid_samples = 32000;
  w.candidate_share = srtb::pipeline::candidate_share(w);
  CHECK(w.candidate_share == 1000);
  w.candidates = {cand(7.25f, 2.5f, 1, 5, 1), cand(12.5f, 3.0f, 8, 999, 40), cand(9.0f, 1.0f, 4, 1000, 2)};
  write_signal_pipe::write_series(w, dir + "/file");
  CHECK(read_text(dir + "/file.1.candidates.csv") ==
        header + "7.25,2.5,1,5,0.32016,1,2,2.75,4,8,3,5\n"
                 "12.5,3,8,999,0.351968,40,2.5,3.25,998,1009,3,998\n");

  // a UDP block (no first sample): share step / 2C = 2048, empty time; the incoherent search's offset S- = 7
  w.first_sample = w.no_first_sample;
  w.valid_samples = 0;
  w.candidate_sample_offset = 7;
  w.candidate_share = srtb::pipeline::candidate_share(w);
  CHECK(w.candidate_share == 2048);
  w.candidates = {cand(6.5f, 0.0f, 2, 2047, 3), cand(8.0f, 4.0f, 1, 2048, 1)};
  write_signal_pipe::write_series(w, dir + "/udp");
  CHECK(read_text(dir + "/udp.1.candidates.csv") == header + "6.5,0,2,2054,,3,-0.5,0.25,2046,2051,3,2046\n");

  // every candidate outside the share: the header row only
  w.candidates = {cand(8.0f, 4.0f, 1, 5000, 1)};
  write_signal_pipe::write_series(w, dir + "/empty");
  CHECK(read_text(dir + "/empty.1.candidates.csv") == header);

  std::printf("candidates ok\n");
  return 0;
}
