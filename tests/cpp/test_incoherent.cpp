// CPU-only tests of the incoherent DM search's host pieces: the incoherent_dm_list config key and its conflict with
// dm_list (include/srtb/program_options.hpp), the block overlap it needs (nsamps_reserved_max in
// include/srtb/pipeline/dedisperse_pipe.hpp) and read_file_pipe's block offsets under it. Links libsrtb_b200.so for its
// host arithmetic (srtb_b200_incoherent_shifts, srtb_b200_nsamps_reserved) and needs no GPU.
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <string>
#include <vector>

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

// the message of what applying `changed` throws, or "" when it does not
static std::string rejection(const std::map<std::string, std::string>& changed) {
  srtb::configs c;
  try {
    srtb::program_options::apply_changed_configs(changed, c);
  } catch (const std::invalid_argument& e) {
    return e.what();
  }
  return "";
}

static unsigned char pattern(size_t i) { return static_cast<unsigned char>(i % 251); }

int main(int argc, char** argv) {
  using srtb::program_options::parse_dm_list;
  srtb::log::current_level = srtb::log::levels::WARNING;
  const std::string dir = (argc > 1) ? argv[1] : "/tmp";

  // ---- the key: the dm_list syntax, from a .cfg line and from the command line
  {
    srtb::configs c;
    srtb::program_options::apply_changed_configs(
        srtb::program_options::parse_config_text("incoherent_dm_list = 9.5:10.5:0.25, 2 * 6\n"), c);
    CHECK(c.incoherent_dm_list == "9.5:10.5:0.25, 2 * 6" && c.dm_list.empty());
    CHECK((parse_dm_list(c.incoherent_dm_list) == std::vector<srtb::real>{9.5f, 9.75f, 10.f, 10.25f, 10.5f, 12.f}));
    std::string a0 = "prog", a1 = "--incoherent_dm_list", a2 = "1:3:1", a3 = "--config_file_name", a4 = dir + "/none.cfg";
    char* av[] = {a0.data(), a1.data(), a2.data(), a3.data(), a4.data()};
    srtb::configs c2;
    srtb::program_options::apply_changed_configs(srtb::program_options::parse_arguments(5, av, "none.cfg"), c2);
    CHECK(c2.incoherent_dm_list == "1:3:1" && parse_dm_list(c2.incoherent_dm_list).size() == 3);
  }
  // a bad list is rejected, naming its key
  for (const char* bad : {"0:1:0", "1,,2", "foo", "1:2", "1:0:0.1"})
    CHECK(rejection({{"incoherent_dm_list", bad}}).find("incoherent_dm_list") != std::string::npos);
  // together with dm_list: rejected, both keys named; either alone is accepted
  {
    const std::string e = rejection({{"dm_list", "0:10:5"}, {"incoherent_dm_list", "1, 2"}});
    CHECK(e.find("dm_list and incoherent_dm_list") != std::string::npos);
    CHECK(rejection({{"dm_list", "0:10:5"}}).empty() && rejection({{"incoherent_dm_list", "1, 2"}}).empty());
    CHECK(rejection({{"dm_list", ""}, {"incoherent_dm_list", "1, 2"}}).empty());
  }

  // ---- the block overlap: nsamps_reserved() + 2C (S+ + S-) when baseband_reserve_sample is set
  auto& cfg = srtb::config;
  cfg.baseband_input_count = 1 << 16;
  cfg.baseband_input_bits = 8;
  cfg.baseband_format_type = "simple";
  cfg.spectrum_channel_count = 16;
  cfg.baseband_sample_rate = 1e8f;
  cfg.baseband_freq_low = 1000.f;
  cfg.baseband_bandwidth = 500.f;
  cfg.baseband_reserve_sample = true;
  cfg.dm = 2e-3f;
  cfg.dm_list = "";
  cfg.incoherent_dm_list = "";
  const size_t base = srtb::codd::nsamps_reserved();
  CHECK(base > 0 && srtb::codd::nsamps_reserved_max() == base);
  cfg.incoherent_dm_list = "1e-3:3e-3:5e-4";
  const std::vector<srtb::real> dms = parse_dm_list(cfg.incoherent_dm_list);
  uint64_t sp = 0, sm = 0;
  CHECK(srtb_b200_incoherent_shifts(16, cfg.baseband_freq_low, cfg.baseband_bandwidth, cfg.baseband_sample_rate,
                                    cfg.dm, dms.data(), dms.size(), nullptr, &sp, &sm) == 0);
  CHECK(sp > 0 && sm > 0);  // trials on both sides of dm
  CHECK(srtb::codd::incoherent_span() == sp + sm);
  const size_t with_inc = srtb::codd::nsamps_reserved_max();
  CHECK(with_inc == base + 2 * 16 * (sp + sm) && with_inc < cfg.baseband_input_count);
  CHECK(srtb::codd::nsamps_reserved() == base);  // unchanged
  {
    std::vector<int64_t> tab(dms.size() * 16);
    uint64_t sp2 = 0, sm2 = 0;
    CHECK(srtb_b200_incoherent_shifts(16, cfg.baseband_freq_low, cfg.baseband_bandwidth, cfg.baseband_sample_rate,
                                      cfg.dm, dms.data(), dms.size(), tab.data(), &sp2, &sm2) == 0);
    CHECK(sp2 == sp && sm2 == sm);
    for (size_t c = 0; c < 16; c++) CHECK(tab[2 * 16 + c] == 0);  // the trial at dm itself
    CHECK(tab[0] < 0 && tab[4 * 16] > 0);                          // below dm reads earlier, above later
  }
  CHECK(srtb_b200_incoherent_shifts(0, 1000.f, 500.f, 1e8f, 0.f, dms.data(), 1, nullptr, nullptr, nullptr) ==
        SRTB_B200_E_INVALID);
  // no reservation asked for: no overlap, as without the list
  cfg.baseband_reserve_sample = false;
  CHECK(srtb::codd::nsamps_reserved_max() == 0);
  cfg.baseband_reserve_sample = true;

  // ---- read_file_pipe's block offsets on a three-block file: each block starts `block - overlap` bytes after the last
  {
    const size_t block = cfg.baseband_input_count, step = block - with_inc;
    const std::string path = dir + "/incoherent_reader.bin";
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
  }
  // the entries are part of the library's ABI
  CHECK(&srtb_b200_incoherent_dm_search != nullptr && &srtb_b200_incoherent_shifts != nullptr);
  std::printf("incoherent ok\n");
  return 0;
}
