// CPU-only tests of the fold's host pieces: the fold_* config keys from a .cfg and the command line and their start-up
// rejections (include/srtb/program_options.hpp), the block timing read_file_pipe stamps on its works (first_sample,
// valid_samples), and the sink's fold_accumulator (include/srtb/pipeline/fold_pipe.hpp): the same file bytes whatever
// order the blocks arrive in. Links libsrtb_b200.so for its host arithmetic and needs no GPU.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <filesystem>
#include <fstream>
#include <random>
#include <string>
#include <vector>

#include "srtb/pipeline/fold_pipe.hpp"
#include "srtb/pipeline/read_file_pipe.hpp"
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

// the message check_fold throws for this config text, or "" when it accepts it
static std::string rejection(const std::string& text) {
  srtb::configs c;
  srtb::program_options::apply_changed_configs(srtb::program_options::parse_config_text(text), c);
  try {
    srtb::program_options::check_fold(c);
  } catch (const std::invalid_argument& e) {
    return e.what();
  }
  return "";
}

static bool has(const std::string& s, const std::string& word) { return s.find(word) != std::string::npos; }

static std::string bytes(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  return std::string((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}

static unsigned char pattern(size_t i) { return static_cast<unsigned char>((i * 131 + 7) % 251); }

// the works read_file_pipe makes of `path` under the current config
static std::vector<srtb::work::copy_to_device_work> read_all(const std::string& path) {
  srtb::config.input_file_path = path;
  srtb::pipeline::read_file_pipe reader;
  std::vector<srtb::work::copy_to_device_work> out;
  while (auto w = reader(std::stop_token{}, srtb::work::dummy_work{})) out.push_back(*w);
  return out;
}

// blocks of random folds, added to an accumulator in the given order; returns the three files' bytes
static std::vector<std::string> accumulate(const std::string& prefix, size_t subint_blocks,
                                           const std::vector<size_t>& order) {
  srtb::pipeline::fold_parameters p;
  p.period = 0.5;
  p.sample_rate = 1e8;
  p.streams = 2;
  p.channels = 16;
  p.subbands = 4;
  p.bins = 9;
  p.block_step = 4096;
  p.subintegration_blocks = subint_blocks;
  p.prefix = prefix;
  srtb::pipeline::fold_accumulator acc{p};
  for (size_t k : order) {
    std::mt19937_64 rng(1000 + k);
    std::uniform_real_distribution<double> u(0.0, 1e6);
    auto b = std::make_shared<srtb::work::fold_block>();
    b->block_index = k;
    b->first_sample = k * p.block_step;
    b->streams = p.streams;
    b->subbands = p.subbands;
    b->bins = p.bins;
    for (size_t i = 0; i < p.streams * p.subbands * p.bins; i++) b->profile.push_back(u(rng) / 3.0);
    for (size_t i = 0; i < p.bins; i++) b->hits.push_back(rng() % 100);
    for (size_t i = 0; i < p.streams * p.subbands; i++) b->kept.push_back((uint32_t)(rng() % 5));
    acc.add(b);
  }
  acc.finish();
  return {bytes(prefix + "fold.npy"), bytes(prefix + "fold.weights.npy"), bytes(prefix + "fold.json")};
}

int main(int argc, char** argv) {
  srtb::log::current_level = srtb::log::levels::WARNING;
  const std::string dir = (argc > 1) ? argv[1] : "/tmp";

  // ---- the keys and their defaults, from a .cfg line and from the command line
  {
    srtb::configs c;
    CHECK(c.fold_period == 0 && c.fold_period_derivative == 0 && c.fold_bin_count == 256 &&
          c.fold_subband_count == 1 && c.fold_subintegration_blocks == 0);
    srtb::program_options::apply_changed_configs(
        srtb::program_options::parse_config_text("fold_period = 0.0893\nfold_period_derivative = 1.25e-13\n"
                                                 "fold_bin_count = 128\nfold_subband_count = 4\n"
                                                 "fold_subintegration_blocks = 3\n"),
        c);
    CHECK(c.fold_period == 0.0893 && c.fold_period_derivative == 1.25e-13 && c.fold_bin_count == 128 &&
          c.fold_subband_count == 4 && c.fold_subintegration_blocks == 3);
    const std::string cfg_path = dir + "/fold.cfg";
    std::ofstream(cfg_path) << "fold_period = 0.5\nfold_bin_count = 64\n";
    std::string a0 = "prog", a1 = "--fold_period", a2 = "0.25", a3 = "--config_file_name", a4 = cfg_path,
                a5 = "--fold_subband_count=8";
    char* av[] = {a0.data(), a1.data(), a2.data(), a3.data(), a4.data(), a5.data()};
    srtb::configs c2;
    srtb::program_options::apply_changed_configs(srtb::program_options::parse_arguments(6, av, "none.cfg"), c2);
    CHECK(c2.fold_period == 0.25 && c2.fold_bin_count == 64 && c2.fold_subband_count == 8);
  }

  // ---- start-up rejections, only with folding on; each names its keys
  {
    const std::string base = "baseband_input_count = 2 ** 20\nspectrum_channel_count = 1024\n"
                             "baseband_sample_rate = 1e8\ninput_file_path = x.bin\n";  // dt = 20.48 us
    CHECK(rejection(base + "fold_period = 0.01\n").empty());
    CHECK(rejection(base + "fold_period = 0.01\nincoherent_dm_list = 1, 2\nsignal_detect_sum_polarizations = 1\n"
                           "gui_enable = 1\nbaseband_write_all = 1\n").empty());
    CHECK(rejection("fold_bin_count = 0\nfold_subband_count = 7\ndm_list = 1, 2\n").empty());  // off: anything
    const std::string neg = rejection(base + "fold_period = -0.01\n");
    CHECK(has(neg, "fold_period") && has(neg, "positive"));
    const std::string nan = rejection(base + "fold_period = 0.01\nfold_period_derivative = 1e400\n");
    CHECK(has(nan, "fold_period_derivative") && has(nan, "finite"));
    const std::string fast = rejection(base + "fold_period = 40e-6\n");
    CHECK(has(fast, "fold_period") && has(fast, "two spectrum samples") && has(fast, "spectrum_channel_count"));
    CHECK(rejection(base + "fold_period = 41e-6\n").empty());
    const std::string bins0 = rejection(base + "fold_period = 0.01\nfold_bin_count = 0\n");
    CHECK(has(bins0, "fold_bin_count") && has(bins0, "1..4096"));
    CHECK(has(rejection(base + "fold_period = 0.01\nfold_bin_count = 4097\n"), "fold_bin_count"));
    CHECK(rejection(base + "fold_period = 0.01\nfold_bin_count = 4096\n").empty());
    const std::string sub = rejection(base + "fold_period = 0.01\nfold_subband_count = 3\n");
    CHECK(has(sub, "fold_subband_count") && has(sub, "spectrum_channel_count"));
    CHECK(rejection(base + "fold_period = 0.01\nfold_subband_count = 1024\n").empty());
    const std::string dml = rejection(base + "fold_period = 0.01\ndm_list = 1, 2\n");
    CHECK(has(dml, "fold_period") && has(dml, "dm_list"));
    const std::string live = rejection("fold_period = 0.01\n");
    CHECK(has(live, "fold_period") && has(live, "input_file_path"));
  }

  // ---- read_file_pipe's block timing: first_sample = k (N - R), valid_samples from the bytes read
  auto& cfg = srtb::config;
  cfg.baseband_input_count = 1 << 16;
  cfg.spectrum_channel_count = 64;
  cfg.baseband_freq_low = 1000;
  cfg.baseband_bandwidth = 64;
  cfg.baseband_sample_rate = 128e6;
  cfg.dm = 0.02f;
  cfg.baseband_reserve_sample = true;
  struct format_case {
    const char* format;
    int bits;
    size_t streams;
  };
  for (const format_case fc : {format_case{"simple", -8, 1}, format_case{"simple", 2, 1},
                               format_case{"naocpsr_snap1", -8, 2}, format_case{"simple", 4, 1}}) {
    for (const size_t offset : {size_t{0}, size_t{1000}}) {
      cfg.baseband_format_type = fc.format;
      cfg.baseband_input_bits = fc.bits;
      cfg.input_file_offset_bytes = offset;
      const size_t N = cfg.baseband_input_count, R = srtb::codd::nsamps_reserved_max();
      CHECK(R > 0 && R < N && R % (2 * cfg.spectrum_channel_count) == 0);
      CHECK(srtb::pipeline::fold_block_step() == N - R);
      const size_t bits = (size_t)std::abs(fc.bits) * fc.streams;  // bits per sample of every stream
      const size_t block_bytes = N * bits / 8, step_bytes = (N - R) * bits / 8;
      const size_t tail = 3 * step_bytes / 7 / 4 * 4;  // a short last block
      const size_t total = offset + block_bytes + 2 * step_bytes + tail;
      const std::string path = dir + "/fold_reader.bin";
      {
        std::ofstream f(path, std::ios::binary | std::ios::trunc);
        for (size_t i = 0; i < total; i++) f.put(static_cast<char>(pattern(i)));
      }
      const auto works = read_all(path);
      CHECK(works.size() == 4);
      for (size_t k = 0; k < works.size(); k++) {
        CHECK(works[k].first_sample == k * (N - R));
        const size_t want_bytes = k < 3 ? block_bytes : total - offset - 3 * step_bytes;
        CHECK(works[k].valid_samples == want_bytes * 8 / bits);
        const auto* b = reinterpret_cast<const unsigned char*>(works[k].baseband_data.baseband_ptr.get());
        CHECK(b[0] == pattern(offset + k * step_bytes));
      }
      CHECK(works[3].valid_samples < N - R);
      // carried to the works the chain makes of it
      srtb::work::write_signal_work w;
      w.copy_parameter_from(works[2]);
      CHECK(w.first_sample == 2 * (N - R) && w.valid_samples == N);
      srtb::work::write_signal_work m;
      m.move_parameter_from(srtb::work::copy_to_device_work{works[1]});
      CHECK(m.first_sample == N - R);
    }
  }
  CHECK(srtb::work::copy_to_device_work{}.first_sample == srtb::work::copy_to_device_work::no_first_sample);

  // ---- the accumulator: in order and shuffled give the same bytes, across subintegration boundaries and with one
  // subintegration for the whole run
  for (const size_t subint_blocks : {size_t{0}, size_t{2}, size_t{3}}) {
    std::vector<size_t> order(7);
    for (size_t i = 0; i < order.size(); i++) order[i] = i;
    const auto ref = accumulate(dir + "/in_order_", subint_blocks, order);
    for (unsigned seed = 1; seed <= 3; seed++) {
      std::mt19937 g(seed);
      std::shuffle(order.begin(), order.end(), g);
      const auto got = accumulate(dir + "/shuffled_" + std::to_string(seed) + "_", subint_blocks, order);
      CHECK(got == ref);
    }
    const size_t subints = subint_blocks ? (7 + subint_blocks - 1) / subint_blocks : 1;
    CHECK(ref[0].size() == 128 + subints * 2 * 4 * 9 * sizeof(double));  // header + [subint][2][4][9] float64
    CHECK(has(ref[2], "\"blocks_folded\": 7") && !std::filesystem::exists(dir + "/in_order_fold.npy.tmp"));
  }
  std::printf("fold ok\n");
  return 0;
}
