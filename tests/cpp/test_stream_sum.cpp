// CPU-only tests of the total-intensity detector's host pieces: the signal_detect_sum_polarizations key from a .cfg
// line and the command line, its three start-up rejections (a single-stream format, dm_list, incoherent_dm_list), and
// write_signal_pipe's keep rule and .sum.<boxcar>.tim files on synthetic works. No GPU: the device calls a cuda_queue
// makes at construction are stood in for below.
#include <cstdio>
#include <cstdlib>
#include <filesystem>
#include <fstream>
#include <string>
#include <vector>

#include "srtb/pipeline/read_file_pipe.hpp"  // backend_registry::get_data_stream_count
#include "srtb/pipeline/write_signal_pipe.hpp"
#include "srtb/program_options.hpp"

// a cuda_queue without a device: no stream, no context
extern "C" cudaError_t cudaSetDevice(int) { return cudaSuccess; }
extern "C" cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) {
  *s = nullptr;
  return cudaSuccess;
}
extern "C" int srtb_b200_ctx_create(int, void*, srtb_b200_ctx** out) {
  *out = nullptr;
  return 0;
}
extern "C" int srtb_b200_ctx_destroy(srtb_b200_ctx*) { return 0; }
extern "C" const char* srtb_b200_last_error(const srtb_b200_ctx*) { return ""; }

#define CHECK(...)                                                                             \
  do {                                                                                         \
    if (!(__VA_ARGS__)) {                                                                      \
      std::fprintf(stderr, "CHECK failed: %s (%s:%d)\n", #__VA_ARGS__, __FILE__, __LINE__); \
      return 1;                                                                                \
    }                                                                                          \
  } while (0)

// the message check_sum_polarizations throws for this config text, or "" when it accepts it
static std::string rejection(const std::string& text) {
  srtb::configs c;
  srtb::program_options::apply_changed_configs(srtb::program_options::parse_config_text(text), c);
  try {
    srtb::program_options::check_sum_polarizations(
        c, srtb::io::backend_registry::get_data_stream_count(c.baseband_format_type));
  } catch (const std::invalid_argument& e) {
    return e.what();
  }
  return "";
}

static srtb::work::time_series_holder series(size_t boxcar, std::vector<float> v) {
  srtb::work::time_series_holder h;
  h.boxcar_length = boxcar;
  h.time_series_length = v.size();
  h.signal_count = 1;
  auto p = std::shared_ptr<srtb::real>(new srtb::real[v.size()], std::default_delete<srtb::real[]>());
  std::copy(v.begin(), v.end(), p.get());
  h.h_time_series = p;
  return h;
}

static std::vector<float> read_floats(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  std::vector<float> v;
  float x;
  while (f.read(reinterpret_cast<char*>(&x), sizeof x)) v.push_back(x);
  return v;
}

int main(int argc, char** argv) {
  srtb::log::current_level = srtb::log::levels::WARNING;
  const std::string dir = (argc > 1) ? argv[1] : "/tmp";

  // ---- the key, from a .cfg line and from the command line (default off)
  {
    srtb::configs c;
    CHECK(!c.signal_detect_sum_polarizations);
    srtb::program_options::apply_changed_configs(
        srtb::program_options::parse_config_text("signal_detect_sum_polarizations = 1\n"), c);
    CHECK(c.signal_detect_sum_polarizations);
    const std::string cfg_path = dir + "/sum.cfg";
    std::ofstream(cfg_path) << "baseband_format_type = naocpsr_snap1\nsignal_detect_sum_polarizations = 0\n";
    std::string a0 = "prog", a1 = "--signal_detect_sum_polarizations", a2 = "1", a3 = "--config_file_name",
                a4 = cfg_path;
    char* av[] = {a0.data(), a1.data(), a2.data(), a3.data(), a4.data()};
    srtb::configs c2;
    srtb::program_options::apply_changed_configs(srtb::program_options::parse_arguments(5, av, "none.cfg"), c2);
    CHECK(c2.signal_detect_sum_polarizations && c2.baseband_format_type == "naocpsr_snap1");
    std::string b1 = "--signal_detect_sum_polarizations=0";
    char* bv[] = {a0.data(), b1.data(), a3.data(), a4.data()};
    srtb::configs c3;
    srtb::program_options::apply_changed_configs(srtb::program_options::parse_arguments(4, bv, "none.cfg"), c3);
    CHECK(!c3.signal_detect_sum_polarizations);
  }

  // ---- start-up rejections
  {
    const std::string on = "signal_detect_sum_polarizations = 1\n";
    CHECK(rejection(on + "baseband_format_type = naocpsr_snap1\n").empty());
    CHECK(rejection(on + "baseband_format_type = gznupsr_a1_4\n").empty());
    CHECK(rejection("baseband_format_type = simple\n").empty());  // key off: any format
    CHECK(rejection("baseband_format_type = simple\ndm_list = 1, 2\n").empty());
    const std::string single = rejection(on + "baseband_format_type = simple\n");
    CHECK(single.find("signal_detect_sum_polarizations") != std::string::npos &&
          single.find("two or more streams") != std::string::npos);
    const std::string dm = rejection(on + "baseband_format_type = naocpsr_snap1\ndm_list = 1, 2\n");
    CHECK(dm.find("signal_detect_sum_polarizations") != std::string::npos && dm.find("dm_list") != std::string::npos);
    const std::string inc = rejection(on + "baseband_format_type = naocpsr_snap1\nincoherent_dm_list = 1, 2\n");
    CHECK(inc.find("signal_detect_sum_polarizations") != std::string::npos &&
          inc.find("incoherent_dm_list") != std::string::npos);
  }

  // ---- the sink: a block whose sum is positive keeps every stream's work; the sum's series are written once
  {
    srtb::config.input_file_path = dir + "/in.bin";  // file mode: only positives are kept
    srtb::config.baseband_output_file_prefix = dir + "/cand_";
    srtb::pipeline::write_signal_pipe sink{srtb::cuda_queue{0}};
    srtb::work::write_signal_work neg;
    neg.timestamp = 7;
    CHECK(!sink.select(neg));
    srtb::work::write_signal_work w0 = neg, w1 = neg;
    w0.sum_positive = w1.sum_positive = true;
    w0.carries_sum = true;
    w0.sum_time_series = {series(1, {1.f, 2.f, 3.f}), series(4, {5.f, 6.f})};
    CHECK(sink.select(w0).has_value());
    CHECK(sink.select(w1).has_value());
    const std::string stem = dir + "/cand_7";
    srtb::pipeline::write_signal_pipe::write_series(w0, stem);
    srtb::pipeline::write_signal_pipe::write_series(w1, stem);
    CHECK((read_floats(stem + ".sum.1.tim") == std::vector<float>{1.f, 2.f, 3.f}));
    CHECK((read_floats(stem + ".sum.4.tim") == std::vector<float>{5.f, 6.f}));
    CHECK(!std::filesystem::exists(stem + ".1.tim") && !std::filesystem::exists(stem + ".4.tim"));
    // a per-stream positive without the sum still writes its own series only
    srtb::work::write_signal_work p = neg;
    p.time_series = {series(2, {9.f})};
    CHECK(sink.select(p).has_value());
    srtb::pipeline::write_signal_pipe::write_series(p, dir + "/cand_8");
    CHECK(std::filesystem::exists(dir + "/cand_8.2.tim") && !std::filesystem::exists(dir + "/cand_8.sum.2.tim"));
  }
  std::printf("stream_sum ok\n");
  return 0;
}
