// srtb/pipeline/write_file_pipe.hpp — the `baseband_write_all` sink (SURVEY §8 f-1): every block's original
// baseband bytes, minus the overlap-save tail the reader re-sends, appended to ONE file named after the first
// block's packet counter (or timestamp). Mirrors the reference's write_file_pipe
// (/root/reference/userspace/include/srtb/pipeline/write_file_pipe.hpp:32-94; selected by
// `baseband_write_all` at /root/reference/userspace/src/main.cpp:206-216). Pure host I/O: the bytes are the
// pinned-host block the work has carried along since the source pipe (work.hpp: baseband_data_holder).
#pragma once
#include <cstdlib>
#include <fstream>
#include <optional>
#include <stdexcept>
#include <stop_token>
#include <string>

#include "srtb/config.hpp"
#include "srtb/cuda_queue.hpp"
#include "srtb/log.hpp"
#include "srtb/pipeline/dedisperse_pipe.hpp"  // srtb::codd::nsamps_reserved
#include "srtb/work.hpp"

namespace srtb {
namespace pipeline {

class write_file_pipe {
 protected:
  std::optional<std::ofstream> opt_file_output_stream;
  std::string file_path;
  srtb::cuda_queue q;

 public:
  explicit write_file_pipe(srtb::cuda_queue q_) : q{q_} {}

  /** path of the file being written ("" before the first work) */
  const std::string& path() const { return file_path; }

  /** accepts what baseband_output_queue carries (write_signal_work slices to write_file_work) */
  std::optional<srtb::work::dummy_work> operator()(std::stop_token, const srtb::work::write_file_work& work) {
    if (!opt_file_output_stream) {
      // the name needs the first block's counter / timestamp, so the file cannot be opened earlier
      auto file_counter = work.udp_packet_counter;
      if (file_counter == work.no_udp_packet_counter) file_counter = work.timestamp;
      file_path = srtb::config.baseband_output_file_prefix + std::to_string(file_counter) + ".bin";
      opt_file_output_stream.emplace(file_path.c_str(), std::ios::binary);
      if (!opt_file_output_stream.value()) {
        const std::string err = "Cannot open file " + file_path;
        SRTB_LOGE << " [write_file_pipe] " << err << srtb::endl;
        opt_file_output_stream.reset();
        throw std::runtime_error{err};
      }
    }
    auto& out = opt_file_output_stream.value();
    const char* ptr = reinterpret_cast<const char*>(work.baseband_data.baseband_ptr.get());
    const size_t input_bytes = work.baseband_data.baseband_input_bytes;
    // the last nsamps_reserved_max() samples come again at the head of the next block
    const size_t nbytes_reserved =
        srtb::codd::nsamps_reserved_max() * static_cast<size_t>(std::abs(srtb::config.baseband_input_bits)) / 8;
    size_t write_bytes = input_bytes;
    if (nbytes_reserved < input_bytes) {
      write_bytes = input_bytes - nbytes_reserved;
      SRTB_LOGD << " [write_file_pipe] " << "reserved " << nbytes_reserved << " bytes" << srtb::endl;
    } else {
      SRTB_LOGW << " [write_file_pipe] " << "baseband_input_bytes = " << input_bytes
                << " <= nbytes_reserved = " << nbytes_reserved << srtb::endl;
    }
    if (ptr && write_bytes) out.write(ptr, static_cast<std::streamsize>(write_bytes));
    if (!out) {
      const std::string err = "Cannot write to " + file_path;
      SRTB_LOGE << " [write_file_pipe] " << err << srtb::endl;
      throw std::runtime_error{err};
    }
    return std::optional{srtb::work::dummy_work{}};
  }
};

}  // namespace pipeline
}  // namespace srtb
