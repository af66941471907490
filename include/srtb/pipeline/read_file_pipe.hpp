// srtb/pipeline/read_file_pipe.hpp — file feeder with overlap-save rewind
// (reference: userspace/include/srtb/pipeline/read_file_pipe.hpp:31-126): each call reads
// baseband_input_count * |bits| / 8 * streams bytes into a zero-filled pinned block, then rewinds the
// file by nsamps_reserved() samples so consecutive blocks overlap by the dispersive smear (:85-99).
// The reference's own H2D copy here duplicates copy_to_device_pipe's (SURVEY q9); this version only
// fills the pinned block — copy_to_device_pipe (or srtb_b200_submit_block) performs the one H2D.
#pragma once
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <optional>
#include <stop_token>

#include "srtb/config.hpp"
#include "srtb/log.hpp"
#include "srtb/memory.hpp"
#include "srtb/pipeline/dedisperse_pipe.hpp"  // srtb::codd::nsamps_reserved
#include "srtb/work.hpp"

namespace srtb {
namespace io {
namespace backend_registry {
/** streams per block of each format (reference: io/backend_registry.hpp:36-181) */
inline size_t get_data_stream_count(const std::string& format) {
  if (format == "naocpsr_snap1" || format == "interleaved_samples_2" || format == "gznupsr_a1") return 2;
  if (format == "gznupsr_a1_4") return 4;
  return 1;
}
}  // namespace backend_registry
}  // namespace io

namespace pipeline {

class read_file_pipe {
 protected:
  std::ifstream input_file_stream;
  std::streamoff logical_file_pos = 0;
  uint64_t block_counter = 0;

 public:
  read_file_pipe() { open(); }
  template <typename Queue>
  explicit read_file_pipe(Queue) { open(); }

  void open() {
    input_file_stream = std::ifstream{srtb::config.input_file_path, std::ifstream::in | std::ifstream::binary};
    input_file_stream.ignore((std::streamsize)srtb::config.input_file_offset_bytes);
    logical_file_pos = (std::streamoff)srtb::config.input_file_offset_bytes;
  }

  std::optional<srtb::work::copy_to_device_work> operator()(std::stop_token, srtb::work::dummy_work) {
    if (!input_file_stream || input_file_stream.peek() == std::ifstream::traits_type::eof()) {
      SRTB_LOGI << " [read_file] " << srtb::config.input_file_path << " has been read";
      return std::nullopt;  // empty optional ends the pipe thread
    }
    const size_t streams = srtb::io::backend_registry::get_data_stream_count(srtb::config.baseband_format_type);
    const size_t time_sample_bytes = srtb::config.baseband_input_count *
                                     static_cast<size_t>(std::abs(srtb::config.baseband_input_bits)) /
                                     srtb::BITS_PER_BYTE * streams;
    auto h_in = srtb::host_allocator.allocate_shared<std::byte>(time_sample_bytes);
    std::memset(h_in.get(), 0, time_sample_bytes);
    // the block's place in the recording, in samples per stream: bytes * 8 / (|bits| * streams)
    const uint64_t bits_per_sample = static_cast<uint64_t>(std::abs(srtb::config.baseband_input_bits)) * streams;
    const uint64_t first_sample =
        (uint64_t)(logical_file_pos - (std::streamoff)srtb::config.input_file_offset_bytes) * srtb::BITS_PER_BYTE /
        bits_per_sample;
    input_file_stream.read(reinterpret_cast<char*>(h_in.get()), (std::streamsize)time_sample_bytes);
    const uint64_t valid_samples = (uint64_t)input_file_stream.gcount() * srtb::BITS_PER_BYTE / bits_per_sample;
    const bool hit_eof = input_file_stream.eof();
    logical_file_pos += (std::streamoff)time_sample_bytes;

    const size_t nsamps_reserved = srtb::codd::nsamps_reserved_max();
    const std::streamoff reserved_bytes =
        (std::streamoff)(nsamps_reserved * static_cast<size_t>(std::abs(srtb::config.baseband_input_bits)) /
                         srtb::BITS_PER_BYTE * streams);
    if (!hit_eof) {
      if (static_cast<size_t>(reserved_bytes) < time_sample_bytes) {
        logical_file_pos -= reserved_bytes;
        input_file_stream.seekg(logical_file_pos);
        SRTB_LOGD << " [read_file] " << "reserved " << reserved_bytes << " bytes";
      } else {
        SRTB_LOGW << " [read_file] " << "time_sample_bytes = " << time_sample_bytes
                  << " >= reserved_bytes = " << reserved_bytes;
      }
    }
    srtb::work::copy_to_device_work w;
    w.ptr = nullptr;  // device copy is made downstream
    w.count = time_sample_bytes;
    w.baseband_data = {h_in, time_sample_bytes};
    w.timestamp = (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(
                      std::chrono::system_clock::now().time_since_epoch())
                      .count();
    w.udp_packet_counter = w.no_udp_packet_counter;
    w.data_stream_id = 0;
    w.first_sample = first_sample;
    w.valid_samples = valid_samples;
    block_counter++;
    return w;
  }
};

}  // namespace pipeline
}  // namespace srtb
