// CPU-only tests of the DM search's host pieces: the dm_list config key (include/srtb/program_options.hpp), the block
// overlap helper and read_file_pipe's block offsets under a dm_list (include/srtb/pipeline/dedisperse_pipe.hpp,
// read_file_pipe.hpp), and the files write_signal_pipe writes for a DM search's work. Links libsrtb_b200.so for its
// host arithmetic (srtb_b200_nsamps_reserved) and needs no GPU: pinned host memory is stood in for below.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>

#include "srtb/pipeline/read_file_pipe.hpp"
#include "srtb/pipeline/write_signal_pipe.hpp"
#include "srtb/program_options.hpp"

// read_file_pipe fills a pinned block from srtb::host_allocator; without a device, plain host memory stands in
extern "C" cudaError_t cudaMallocHost(void** ptr, size_t size) {
  *ptr = std::malloc(size);
  return *ptr ? cudaSuccess : cudaErrorMemoryAllocation;
}
extern "C" cudaError_t cudaFreeHost(void* ptr) {
  std::free(ptr);
  return cudaSuccess;
}

#define CHECK(...)                                                                             \
  do {                                                                                         \
    if (!(__VA_ARGS__)) {                                                                      \
      std::fprintf(stderr, "CHECK failed: %s (%s:%d)\n", #__VA_ARGS__, __FILE__, __LINE__); \
      return 1;                                                                                \
    }                                                                                          \
  } while (0)

static bool rejects(const std::string& list) {
  srtb::configs c;
  try {
    srtb::program_options::apply_changed_configs({{"dm_list", list}}, c);
  } catch (const std::invalid_argument& e) {
    return std::string{e.what()}.find("dm_list") != std::string::npos;  // the key is named
  }
  return false;
}

static std::string read_text(const std::string& path) {
  std::ifstream f(path);
  std::stringstream ss;
  ss << f.rdbuf();
  return ss.str();
}

// the byte at file offset i of the reader test's file
static unsigned char pattern(size_t i) { return static_cast<unsigned char>(i % 251); }

int main(int argc, char** argv) {
  using srtb::program_options::parse_dm_list;
  srtb::log::current_level = srtb::log::levels::WARNING;
  const std::string dir = (argc > 1) ? argv[1] : "/tmp";

  // ---- dm_list parsing: lists, expressions, ranges, order
  CHECK(parse_dm_list("").empty() && parse_dm_list("  ").empty());
  CHECK((parse_dm_list("56.778") == std::vector<srtb::real>{56.778f}));
  CHECK((parse_dm_list("10, 2 * 281.025, -478.80") == std::vector<srtb::real>{10.f, 562.05f, -478.80f}));
  CHECK((parse_dm_list("30, 10, 20") == std::vector<srtb::real>{30.f, 10.f, 20.f}));  // the list's order is kept
  CHECK((parse_dm_list("0:10:5") == std::vector<srtb::real>{0.f, 5.f, 10.f}));
  CHECK((parse_dm_list("0:9:5") == std::vector<srtb::real>{0.f, 5.f, 10.f}));  // floor(9/5 + 0.5) = 2
  CHECK((parse_dm_list("0:7:5") == std::vector<srtb::real>{0.f, 5.f}));        // floor(7/5 + 0.5) = 1
  CHECK((parse_dm_list("5:5:1") == std::vector<srtb::real>{5.f}));
  CHECK((parse_dm_list("2 ** 2 : 2 * 4 : 1 + 1, 100") == std::vector<srtb::real>{4.f, 6.f, 8.f, 100.f}));
  CHECK((parse_dm_list("-10:-5:5") == std::vector<srtb::real>{-10.f, -5.f}));
  {
    const auto v = parse_dm_list("0:1:0.1");  // start + i * step in double: no drift from repeated addition
    CHECK(v.size() == 11 && v.front() == 0.f && v.back() == 1.0f);
    for (size_t i = 0; i < v.size(); i++) CHECK(v[i] == static_cast<srtb::real>(0.0 + (double)i * 0.1));
  }
  for (const char* bad : {"0:1:0", "0:1:-0.5", "1:0:0.1", "1,,2", "1,", ",1", " , ", "foo", "1:x:1", "1:2", "1:2:3:4",
                          "2 **", "0:1e400:1", "(1"})
    CHECK(rejects(bad));
  {
    srtb::configs c;
    srtb::program_options::apply_changed_configs(srtb::program_options::parse_config_text("dm_list = 0:100:50, 7\n"), c);
    CHECK(c.dm_list == "0:100:50, 7" && (parse_dm_list(c.dm_list) == std::vector<srtb::real>{0.f, 50.f, 100.f, 7.f}));
    std::string a0 = "prog", a1 = "--dm_list", a2 = "1:3:1", a3 = "--config_file_name", a4 = dir + "/none.cfg";
    char* av[] = {a0.data(), a1.data(), a2.data(), a3.data(), a4.data()};
    srtb::configs c2;
    srtb::program_options::apply_changed_configs(srtb::program_options::parse_arguments(5, av, "none.cfg"), c2);
    CHECK(c2.dm_list == "1:3:1" && parse_dm_list(c2.dm_list).size() == 3);
  }
  // the reference's two shipped configuration files still load unchanged, with no DM list
  if (argc > 2) {
    for (const char* name : {"/srtb_config.cfg", "/srtb_config_1644-4559.cfg"}) {
      std::string b0 = "prog", b1 = "--config_file_name", b2 = std::string{argv[2]} + name;
      char* bv[] = {b0.data(), b1.data(), b2.data()};
      srtb::configs r;
      srtb::program_options::apply_changed_configs(srtb::program_options::parse_arguments(3, bv, "none.cfg"), r);
      CHECK(r.dm_list.empty() && r.baseband_input_count == (size_t{1} << 30) && r.spectrum_channel_count == 2048);
      CHECK(r.dm == (std::string{name} == "/srtb_config.cfg" ? 0.0f : -478.80f));
    }
    srtb::log::current_level = srtb::log::levels::WARNING;
  }

  // ---- the overlap helper: the largest reserve over the trials, of the function itself
  auto& cfg = srtb::config;
  cfg.baseband_input_count = 8192;
  cfg.baseband_input_bits = 8;
  cfg.baseband_format_type = "simple";
  cfg.spectrum_channel_count = 16;
  cfg.baseband_sample_rate = 1e9f;
  cfg.baseband_reserve_sample = true;
  auto reserved_at = [&](srtb::real dm) {
    return srtb_b200_nsamps_reserved(cfg.baseband_input_count, cfg.spectrum_channel_count, cfg.baseband_freq_low,
                                     cfg.baseband_bandwidth, cfg.baseband_sample_rate, dm, 1);
  };
  // an inverted band (bandwidth < 0) with negative DMs delays, the largest |DM| (positive here) reserves nothing
  cfg.baseband_freq_low = 1500.f;
  cfg.baseband_bandwidth = -500.f;
  cfg.dm = 0;
  cfg.dm_list = "5e-4, -1e-4, 0, -3e-4:-2e-4:1e-4";
  CHECK(reserved_at(5e-4f) == 0 && reserved_at(-1e-4f) > 0 && reserved_at(-3e-4f) > reserved_at(-2e-4f));
  const size_t max_reserved = srtb::codd::nsamps_reserved_max();
  CHECK(max_reserved == reserved_at(-3e-4f) && max_reserved > 0);
  CHECK(srtb::codd::nsamps_reserved() == 0);  // what nsamps_reserved() returns (at dm = 0) is unchanged
  // the normal band: positive DMs delay
  cfg.baseband_freq_low = 1000.f;
  cfg.baseband_bandwidth = 500.f;
  cfg.baseband_reserve_sample = true;
  cfg.dm_list = "-5e-4, 1e-4, 2e-4";
  CHECK(srtb::codd::nsamps_reserved_max() == reserved_at(2e-4f) && reserved_at(2e-4f) > reserved_at(1e-4f));
  // no dm_list: exactly nsamps_reserved() at dm
  cfg.dm_list = "";
  cfg.dm = 3e-4f;
  CHECK(srtb::codd::nsamps_reserved_max() == srtb::codd::nsamps_reserved() && srtb::codd::nsamps_reserved() == reserved_at(3e-4f));

  // ---- read_file_pipe's block offsets on a three-block file: each block starts `block - reserve` bytes after the last
  auto check_reader = [&](size_t reserve) -> int {
    const size_t block = cfg.baseband_input_count, step = block - reserve;
    const std::string path = dir + "/dm_list_reader.bin";
    {
      std::ofstream f(path, std::ios::binary | std::ios::trunc);
      for (size_t i = 0; i < block + 2 * step; i++) f.put(static_cast<char>(pattern(i)));
    }
    cfg.input_file_path = path;
    cfg.input_file_offset_bytes = 0;
    srtb::pipeline::read_file_pipe reader;
    for (size_t k = 0; k < 3; k++) {
      auto w = reader(std::stop_token{}, srtb::work::dummy_work{});
      CHECK(w.has_value() && w->baseband_data.baseband_input_bytes == block);
      const auto* b = reinterpret_cast<const unsigned char*>(w->baseband_data.baseband_ptr.get());
      for (size_t j = 0; j < block; j++) CHECK(b[j] == pattern(k * step + j));
    }
    return 0;
  };
  cfg.baseband_freq_low = 1500.f;
  cfg.baseband_bandwidth = -500.f;
  cfg.baseband_reserve_sample = true;
  cfg.dm = 0;
  cfg.dm_list = "5e-4, -1e-4, 0, -3e-4:-2e-4:1e-4";
  CHECK(check_reader(reserved_at(-3e-4f)) == 0);
  cfg.dm_list = "";  // today's overlap: nsamps_reserved() at dm
  cfg.dm = -2e-4f;
  CHECK(check_reader(reserved_at(-2e-4f)) == 0 && reserved_at(-2e-4f) > 0);

  // ---- write_signal_pipe's files for a DM search's work (host data only: no spectrum pointer)
  {
    srtb::work::write_signal_work w;
    w.data_stream_id = 1;
    w.dm = 12.5f;
    std::vector<float> series(2 * 8);
    for (size_t i = 0; i < series.size(); i++) series[i] = (float)i;
    auto owner = std::shared_ptr<srtb::real>(series.data(), [](srtb::real*) {});
    w.time_series.push_back({owner, 8, 1, 3});
    w.time_series.push_back({std::shared_ptr<srtb::real>(owner, series.data() + 8), 7, 2, 1});
    srtb::work::dm_trial_summary off;
    off.dm = 0;
    off.detect_enabled = false;
    srtb::work::dm_trial_summary on;
    on.dm = 12.5f;
    on.detect_enabled = true;
    on.boxcars.push_back({1, 8, 3, 1.5f, 7.25f, 4});
    on.boxcars.push_back({2, 7, 1, 2.0f, 6.5f, 3});
    w.dm_trials = {off, on};
    const std::string stem = dir + "/cand_42";
    srtb::pipeline::write_signal_pipe::write_series(w, stem);
    std::ifstream t1(stem + ".dm12.5.1.tim", std::ios::binary), t2(stem + ".dm12.5.2.tim", std::ios::binary);
    CHECK(t1.good() && t2.good());
    std::vector<float> r1(8), r2(7);
    t1.read(reinterpret_cast<char*>(r1.data()), 8 * sizeof(float));
    t2.read(reinterpret_cast<char*>(r2.data()), 7 * sizeof(float));
    CHECK(t1.gcount() == 32 && t2.gcount() == 28 && r1[7] == 7.f && r2[0] == 8.f && r2[6] == 14.f);
    CHECK(read_text(stem + ".1.dm_sweep.csv") ==
          "dm,detect_enabled,boxcar_length,series_length,signal_count,threshold,peak_snr,peak_index\n"
          "0,0,0,0,0,0,0,0\n"
          "12.5,1,1,8,3,1.5,7.25,4\n"
          "12.5,1,2,7,1,2,6.5,3\n");
    // a work without dm_trials is written as before: <stem>.<boxcar>.tim, no table
    srtb::work::write_signal_work plain;
    plain.time_series.push_back({owner, 8, 4, 1});
    srtb::pipeline::write_signal_pipe::write_series(plain, stem);
    CHECK(std::ifstream(stem + ".4.tim").good() && !std::ifstream(stem + ".0.dm_sweep.csv").good());
  }
  // the DM search entry is part of the library's ABI
  CHECK(&srtb_b200_process_block_dm_sweep_ex != nullptr);
  std::printf("dm list ok\n");
  return 0;
}
