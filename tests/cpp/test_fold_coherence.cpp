// CPU-only tests of the folded coherence products' host pieces: the fold_coherence key from a .cfg and the command line
// and its start-up rejections (include/srtb/program_options.hpp), and the sink's fold_accumulator
// (include/srtb/pipeline/fold_pipe.hpp) with the key on: block-order sums whatever order the blocks arrive in, the
// coherence files' shapes and weights, and the plain fold's files unchanged by the key. Links libsrtb_b200.so for its
// host arithmetic and needs no GPU.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <filesystem>
#include <fstream>
#include <random>
#include <string>
#include <vector>

#include "srtb/pipeline/fold_pipe.hpp"
#include "srtb/program_options.hpp"

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

// the float64 payload of a .npy file (its header is 128 bytes for these shapes)
static std::vector<double> npy_values(const std::string& path) {
  const std::string b = bytes(path);
  std::vector<double> v((b.size() - 128) / sizeof(double));
  std::memcpy(v.data(), b.data() + 128, v.size() * sizeof(double));
  return v;
}

constexpr size_t STREAMS = 2, SUBBANDS = 4, BINS = 9, BLOCKS = 7;

static srtb::pipeline::fold_parameters parameters(const std::string& prefix, size_t subint_blocks, bool coherence) {
  srtb::pipeline::fold_parameters p;
  p.period = 0.5;
  p.sample_rate = 1e8;
  p.streams = STREAMS;
  p.channels = 16;
  p.subbands = SUBBANDS;
  p.bins = BINS;
  p.block_step = 4096;
  p.subintegration_blocks = subint_blocks;
  p.coherence = coherence;
  p.prefix = prefix;
  return p;
}

// block k's fold: random profile, hits and kept, and (with coherence) random products and kept-in-both counts
static std::shared_ptr<srtb::work::fold_block> block(size_t k, bool coherence) {
  std::mt19937_64 rng(1000 + k);
  std::uniform_real_distribution<double> u(-1e6, 1e6);
  auto b = std::make_shared<srtb::work::fold_block>();
  b->block_index = k;
  b->first_sample = k * 4096;
  b->streams = STREAMS;
  b->subbands = SUBBANDS;
  b->bins = BINS;
  for (size_t i = 0; i < STREAMS * SUBBANDS * BINS; i++) b->profile.push_back(std::abs(u(rng)) / 3.0);
  for (size_t i = 0; i < BINS; i++) b->hits.push_back(rng() % 100);
  for (size_t i = 0; i < STREAMS * SUBBANDS; i++) b->kept.push_back((uint32_t)(rng() % 5));
  if (coherence) {
    for (size_t i = 0; i < 4 * SUBBANDS * BINS; i++) b->coherence.push_back(u(rng) / 7.0);
    for (size_t i = 0; i < SUBBANDS; i++) b->coherence_kept.push_back((uint32_t)(rng() % 4));
  }
  return b;
}

static const char* const FILES[] = {"fold.npy", "fold.weights.npy", "fold.json", "fold.coherence.npy",
                                    "fold.coherence.weights.npy"};

// the blocks added in `order`; returns the five files' bytes ("" for a file not written)
static std::vector<std::string> accumulate(const std::string& prefix, size_t subint_blocks,
                                           const std::vector<size_t>& order, bool coherence) {
  srtb::pipeline::fold_accumulator acc{parameters(prefix, subint_blocks, coherence)};
  for (size_t k : order) acc.add(block(k, coherence));
  acc.finish();
  std::vector<std::string> out;
  for (const char* f : FILES) out.push_back(std::filesystem::exists(prefix + f) ? bytes(prefix + f) : "");
  return out;
}

int main(int argc, char** argv) {
  srtb::log::current_level = srtb::log::levels::WARNING;
  const std::string dir = (argc > 1) ? argv[1] : "/tmp";

  // ---- the key and its default, from a .cfg line and from the command line
  {
    srtb::configs c;
    CHECK(!c.fold_coherence);
    srtb::program_options::apply_changed_configs(srtb::program_options::parse_config_text("fold_coherence = 1\n"), c);
    CHECK(c.fold_coherence);
    std::string a0 = "prog", a1 = "--fold_coherence", a2 = "1";
    char* av[] = {a0.data(), a1.data(), a2.data()};
    srtb::configs c2;
    srtb::program_options::apply_changed_configs(srtb::program_options::parse_arguments(3, av, "none.cfg"), c2);
    CHECK(c2.fold_coherence);
  }

  // ---- start-up rejections; each names the key
  {
    const std::string base = "baseband_input_count = 2 ** 20\nspectrum_channel_count = 1024\n"
                             "baseband_sample_rate = 1e8\ninput_file_path = x.bin\n";
    const std::string on = base + "fold_period = 0.01\nfold_coherence = 1\n";
    for (const char* f : {"naocpsr_snap1", "interleaved_samples_2", "gznupsr_a1"})
      CHECK(rejection(on + "baseband_format_type = " + f + "\n").empty());
    const std::string no_period = rejection(base + "fold_coherence = 1\nbaseband_format_type = naocpsr_snap1\n");
    CHECK(has(no_period, "fold_coherence") && has(no_period, "fold_period"));
    for (const char* f : {"simple", "fastmb_roach2", "naocpsr_roach2"}) {
      const std::string single = rejection(on + "baseband_format_type = " + f + "\n");
      CHECK(has(single, "fold_coherence") && has(single, "single-stream"));
    }
    const std::string four = rejection(on + "baseband_format_type = gznupsr_a1_4\n");
    CHECK(has(four, "fold_coherence") && has(four, "gznupsr_a1_4"));
    // off: the plain fold's checks alone
    CHECK(rejection(base + "fold_period = 0.01\nfold_coherence = 0\nbaseband_format_type = gznupsr_a1_4\n").empty());
  }

  // ---- the accumulator with the key on: in order and shuffled give the same bytes; the sums, shapes and weights
  for (const size_t subint_blocks : {size_t{0}, size_t{2}, size_t{3}}) {
    std::vector<size_t> order(BLOCKS);
    for (size_t i = 0; i < order.size(); i++) order[i] = i;
    const std::string pre = dir + "/coh_" + std::to_string(subint_blocks) + "_";
    const auto ref = accumulate(pre + "in_order_", subint_blocks, order, true);
    for (unsigned seed = 1; seed <= 3; seed++) {
      std::mt19937 g(seed);
      std::shuffle(order.begin(), order.end(), g);
      CHECK(accumulate(pre + "shuffled_" + std::to_string(seed) + "_", subint_blocks, order, true) == ref);
    }
    const size_t subints = subint_blocks ? (BLOCKS + subint_blocks - 1) / subint_blocks : 1;
    CHECK(ref[3].size() == 128 + subints * 4 * SUBBANDS * BINS * sizeof(double));
    CHECK(ref[4].size() == 128 + subints * SUBBANDS * BINS * sizeof(double));
    CHECK(has(ref[3].substr(0, 128), "(" + std::to_string(subints) + ", 4, 4, 9)"));
    CHECK(has(ref[4].substr(0, 128), "(" + std::to_string(subints) + ", 4, 9)"));
    CHECK(has(ref[2], "\"coherence\": [\"AA\", \"BB\", \"CR\", \"CI\"]") && has(ref[2], "X = stream 0") &&
          has(ref[2], "no calibration"));
    // block-order float64 sums, and weights = sum over blocks of kept-in-both[k] hits[bin]
    std::vector<double> coh(subints * 4 * SUBBANDS * BINS, 0.0), wts(subints * SUBBANDS * BINS, 0.0);
    for (size_t k = 0; k < BLOCKS; k++) {
      const auto b = block(k, true);
      const size_t si = subint_blocks ? k / subint_blocks : 0;
      for (size_t i = 0; i < 4 * SUBBANDS * BINS; i++) coh[si * 4 * SUBBANDS * BINS + i] += b->coherence[i];
      for (size_t s = 0; s < SUBBANDS; s++)
        for (size_t bin = 0; bin < BINS; bin++)
          wts[(si * SUBBANDS + s) * BINS + bin] += (double)b->coherence_kept[s] * (double)b->hits[bin];
    }
    CHECK(npy_values(pre + "in_order_fold.coherence.npy") == coh);
    CHECK(npy_values(pre + "in_order_fold.coherence.weights.npy") == wts);
    CHECK(!std::filesystem::exists(pre + "in_order_fold.coherence.npy.tmp"));

    // the key off: no coherence files, and the plain fold's files are those of the key on, less the coherence lines
    const auto off = accumulate(pre + "off_", subint_blocks, order, false);
    CHECK(off[3].empty() && off[4].empty());
    CHECK(off[0] == ref[0] && off[1] == ref[1]);
    CHECK(!has(off[2], "coherence"));
    std::string json_on = ref[2];
    const size_t a = json_on.find("  \"coherence\""), e = json_on.find("  \"reference\"");
    CHECK(a != std::string::npos && e != std::string::npos && a < e);
    CHECK(json_on.erase(a, e - a) == off[2]);
  }

  // ---- a block without the products in a run that has the key on is refused
  {
    srtb::pipeline::fold_accumulator acc{parameters(dir + "/refuse_", 0, true)};
    bool threw = false;
    try {
      acc.add(block(0, false));
    } catch (const std::runtime_error&) {
      threw = true;
    }
    CHECK(threw);
  }
  std::printf("fold coherence ok\n");
  return 0;
}
