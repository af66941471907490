// CPU-only tests of the candidate cut-outs' host pieces: the candidate_cutouts key (include/srtb/program_options.hpp) in
// a .cfg and on the command line and its start-up refusals, the top-N selection and its ties, the plane's DM half-width
// and the requests (include/srtb/pipeline/baseband_chain_pipe.hpp), and the exact <stem>.<id>.cutouts.csv and .npy
// shapes write_signal_pipe writes for a hand-made work. Links libsrtb_b200.so and needs no GPU.
#include <cmath>
#include <cstdio>
#include <filesystem>
#include <fstream>
#include <sstream>
#include <string>

#include "srtb/pipeline/baseband_chain_pipe.hpp"
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
  std::ifstream f(path, std::ios::binary);
  std::stringstream ss;
  ss << f.rdbuf();
  return ss.str();
}

static srtb::work::dm_candidate cand(float snr, float dm, uint64_t boxcar, uint64_t window) {
  srtb::work::dm_candidate c;
  c.snr = snr;
  c.dm = dm;
  c.dm_low = c.dm_high = dm;
  c.boxcar_length = boxcar;
  c.window = window;
  c.peak_index = window;
  c.members = 1;
  return c;
}

// the message of check_candidate_cutouts' refusal, or "" when it accepts c
static std::string refusal(const srtb::configs& c) {
  try {
    srtb::program_options::check_candidate_cutouts(c);
  } catch (const std::invalid_argument& e) {
    return e.what();
  }
  return "";
}

int main(int argc, char** argv) {
  srtb::log::current_level = srtb::log::levels::WARNING;
  const std::string dir = (argc > 1) ? argv[1] : "/tmp";
  using srtb::program_options::apply_changed_configs;

  // ---- the key, in a .cfg and on the command line, and the start-up refusals
  {
    srtb::configs c;
    CHECK(c.candidate_cutouts == 0);
    CHECK(refusal(c).empty());
    apply_changed_configs(srtb::program_options::parse_config_text("candidate_cutouts = 4\n"), c);
    CHECK(c.candidate_cutouts == 4);
    apply_changed_configs({{"candidate_cutouts", "2 * 3"}}, c);  // the command line's value, an expression
    CHECK(c.candidate_cutouts == 6);
    std::string m = refusal(c);  // no candidate list
    CHECK(m.find("candidate_cutouts") != std::string::npos && m.find("signal_detect_candidates") != std::string::npos &&
          m.find("dm_search_candidates") != std::string::npos);
    c.signal_detect_candidates = true;
    CHECK(refusal(c).empty());
    c.signal_detect_candidates = false;
    c.dm_search_candidates = true;
    c.incoherent_dm_list = "1, 2";
    CHECK(refusal(c).empty());
    c.incoherent_dm_list = "";
    c.dm_list = "1, 2";
    m = refusal(c);  // the coherent sweep keeps no trial's spectrum
    CHECK(m.find("candidate_cutouts") != std::string::npos && m.find("dm_list") != std::string::npos);
    c.dm_list = "";
    apply_changed_configs({{"candidate_cutouts", "-1"}}, c);
    CHECK(c.candidate_cutouts == -1);
    m = refusal(c);
    CHECK(m.find("candidate_cutouts") != std::string::npos && m.find("-1") != std::string::npos);
    apply_changed_configs({{"candidate_cutouts", "0"}}, c);
    c.dm_list = "1, 2";
    CHECK(refusal(c).empty());  // off: nothing to refuse
    bool known = true;
    try {
      srtb::program_options::check_known("candidate_cutouts");
    } catch (...) {
      known = false;
    }
    CHECK(known);
  }

  // ---- the fixed geometry: nsub is the largest divisor of C up to 256
  CHECK(srtb::pipeline::cutout_nsub(2048) == 256);
  CHECK(srtb::pipeline::cutout_nsub(256) == 256);
  CHECK(srtb::pipeline::cutout_nsub(16) == 16);
  CHECK(srtb::pipeline::cutout_nsub(1000) == 250);
  CHECK(srtb::pipeline::cutout_nsub(257) == 1);
  CHECK(srtb::pipeline::cutout_nsub(1) == 1);

  // ---- the half-width: the DM offset whose residual sweep across the band fills half the image
  {
    const size_t C = 2048;
    const float fl = 1000.f, bw = 500.f, sr = 4e9f;
    const double k_max = srtb::pipeline::cutout_k_max(C, fl, bw, sr);
    // the lowest channel's delay, the largest (f_ref is the top edge for a positive bandwidth)
    const double f0 = (double)fl + (double)bw * 0.5 / (double)C, fr = (double)(float)(fl + bw);
    const double k0 = (1.0 / (f0 * f0) - 1.0 / (fr * fr)) * ((double)sr / (2.0 * C)) * 4.148808e3;
    CHECK(k_max == std::fabs(k0));
    // the same band read downward: f_ref the bottom edge, so the largest delay is the top channel's
    const double k_dn = srtb::pipeline::cutout_k_max(C, 1500.f, -500.f, sr);
    CHECK(k_dn > 0 && std::fabs(k_dn - k_max) < 0.01 * k_max);
    for (uint32_t q : {1u, 3u, 16u, 128u}) {
      const float hw = srtb::pipeline::cutout_halfwidth(256, q, k_max);
      CHECK(hw == (float)(128.0 * q / k_max));
      CHECK(std::fabs((double)hw * k_max / q - 128.0) < 1e-3);  // the sweep at the plane's edge row: W/2 bins
    }
    CHECK(srtb::pipeline::cutout_halfwidth(256, 4, 0.0) == 0.f);
  }

  // ---- the selection: the N highest-S/N rows of the file (window below the share), ties in file order
  {
    std::vector<srtb::work::dm_candidate> cs = {cand(7, 10, 4, 100), cand(9, 11, 1, 200), cand(7, 12, 2, 5000),
                                                cand(8, 10, 8, 300), cand(7, 13, 16, 400), cand(12, 14, 32, 9000)};
    // cs[2] and cs[5] lie past the share of 1000: not in the file, so never cut out. File rows: 0 1 2 3 = cs 0 1 3 4
    auto sel = srtb::pipeline::cutout_selection(cs, 1000, 3);
    CHECK(sel.size() == 3);
    CHECK(sel[0].first == 1 && sel[0].second == 1);  // S/N 9
    CHECK(sel[1].first == 2 && sel[1].second == 3);  // S/N 8
    CHECK(sel[2].first == 0 && sel[2].second == 0);  // S/N 7, the first of the tie in file order
    sel = srtb::pipeline::cutout_selection(cs, 1000, 10);
    CHECK(sel.size() == 4 && sel[3].first == 3 && sel[3].second == 4);
    CHECK(srtb::pipeline::cutout_selection(cs, 50, 4).empty());
    // the requests: q = max(1, boxcar / 2), center = window + offset + boxcar / 2, the candidate's DM
    const auto req = srtb::pipeline::cutout_requests(cs, sel, 17, 1000.0);
    CHECK(req.size() == 4);
    CHECK(req[0].decimation == 1 && req[0].center == 200 + 17 + 0 && req[0].dm == 11.f);
    CHECK(req[1].decimation == 4 && req[1].center == 300 + 17 + 4 && req[1].dm == 10.f);
    CHECK(req[2].decimation == 2 && req[2].center == 100 + 17 + 2);
    CHECK(req[3].decimation == 8 && req[3].center == 400 + 17 + 8 && req[3].dm == 13.f);
    CHECK(req[1].dm_halfwidth == srtb::pipeline::cutout_halfwidth(256, 4, 1000.0));
  }

  // ---- the files: exact csv text, npy shapes, the sum's names, and an empty time without a first sample
  {
    srtb::config.baseband_sample_rate = 4e9;
    srtb::work::write_signal_work w;
    w.batch_size = 2048;
    w.data_stream_id = 1;
    w.first_sample = 1000;
    auto c = std::make_shared<srtb::work::cutout_set>();
    c->width = 4;
    c->nsub = 2;
    c->n_rows = 3;
    c->ft.assign(2 * 2 * 4, 1.5f);
    c->dmt.assign(2 * 3 * 4, 2.5f);
    c->rows.push_back({2, 5000, 1, 9.5f, 10.5f});
    c->rows.push_back({0, 3, 16, 0.25f, 1.75f});
    const std::string stem = dir + "/cut";
    srtb::pipeline::write_signal_pipe::write_cutouts(w, *c, stem + ".1");
    const std::string want =
        "candidate,center,decimation,time,dm_row_low,dm_row_high\n"
        "2,5000,1,0.005118202,9.5,10.5\n"  // bin 0 at 4998: (1000 + 4096 * 4998) / 4e9
        "0,3,16,-2.9446e-05,0.25,1.75\n";  // bin 0 at 3 - 2 * 16 = -29
    const std::string got = read_text(stem + ".1.cutouts.csv");
    if (got != want) std::fprintf(stderr, "got:\n%s", got.c_str());
    CHECK(got == want);
    const std::string ft = read_text(stem + ".1.cutout_ft.npy");
    const std::string dmt = read_text(stem + ".1.cutout_dmt.npy");
    CHECK(ft.find("'descr': '<f4'") != std::string::npos && ft.find("(2, 2, 4)") != std::string::npos);
    CHECK(dmt.find("(2, 3, 4)") != std::string::npos);
    w.first_sample = w.no_first_sample;
    srtb::pipeline::write_signal_pipe::write_cutouts(w, *c, stem + ".sum");
    CHECK(read_text(stem + ".sum.cutouts.csv") ==
          "candidate,center,decimation,time,dm_row_low,dm_row_high\n2,5000,1,,9.5,10.5\n0,3,16,,0.25,1.75\n");
  }
  std::printf("cutouts ok\n");
  return 0;
}
