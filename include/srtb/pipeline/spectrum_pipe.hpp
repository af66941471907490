// srtb/pipeline/spectrum_pipe.hpp — simplify_spectrum_pipe_2 (reference: pipeline/spectrum_pipe.hpp:82-143): a block's
// dynamic spectrum -> gui_pixmap_width x gui_pixmap_height ARGB32 thumbnail (srtb_b200_simplify_spectrum: three
// kernels, see csrc/thumbnail.cuh), copied to the host; plus the headless sink that shows it, one binary PPM per data
// stream replaced atomically on every block (the counterpart of the reference's refreshed Qt window).
#pragma once
#include <atomic>
#include <cstdint>
#include <cstdio>
#include <filesystem>
#include <fstream>
#include <optional>
#include <stop_token>
#include <string>
#include <vector>

#include "srtb/config.hpp"
#include "srtb/cuda_queue.hpp"
#include "srtb/log.hpp"
#include "srtb/memory.hpp"
#include "srtb/work.hpp"

namespace srtb {
namespace pipeline {

/** the thumbnail side branch of one GPU (main.cpp:197-201 of the reference): each block is pushed once into a bounded
 *  queue and dropped when the queue is full, like the reference's loose_queue_out_functor on its capacity-2 queue, so
 *  a busy thumbnail pipe makes the branch skip blocks instead of holding their spectra. Closed until `open` is set (the
 *  start-up warm-up blocks leave no thumbnail). `accepted` / `dropped` count the blocks that entered the queue / that
 *  found it full. The host baseband of the block is not carried along. */
struct thumbnail_out_functor {
  using queue = srtb::bounded_mpmc_queue<srtb::work::simplify_spectrum_work>;
  std::shared_ptr<queue> q;
  std::shared_ptr<std::atomic<bool>> open;
  std::shared_ptr<std::atomic<uint64_t>> accepted = std::make_shared<std::atomic<uint64_t>>(0);
  std::shared_ptr<std::atomic<uint64_t>> dropped = std::make_shared<std::atomic<uint64_t>>(0);
  template <typename Work>
  void operator()(std::stop_token st, const Work& w) {
    if (st.stop_requested() || !open->load()) return;
    srtb::work::simplify_spectrum_work t = w;  // a write_signal_work converts: the device spectrum and its identity
    t.baseband_data = {};
    if (q->push(t)) (*accepted)++;
    else (*dropped)++;
  }
};

class simplify_spectrum_pipe_2 {
 public:
  srtb::cuda_queue q;
  explicit simplify_spectrum_pipe_2(srtb::cuda_queue q_) : q{q_} {}

  /** a write_signal_work (the chain's output) converts to simplify_spectrum_work */
  std::optional<srtb::work::draw_spectrum_work_2> operator()(std::stop_token,
                                                             srtb::work::simplify_spectrum_work w) {
    cuda_check(cudaSetDevice(q.device()), "cudaSetDevice");
    const size_t in_width = w.count, in_height = w.batch_size;
    const size_t out_width = srtb::config.gui_pixmap_width, out_height = srtb::config.gui_pixmap_height;
    const size_t n = out_width * out_height;
    auto d_intensity = srtb::device_allocator.allocate_shared<srtb::real>(n);
    auto d_image = srtb::device_allocator.allocate_shared<uint32_t>(n);
    auto h_image = srtb::host_allocator.allocate_shared<uint32_t>(n);
    q.check(srtb_b200_simplify_spectrum(q.ctx(), w.ptr.get(), in_width, in_height, out_width, out_height,
                                        srtb::gui::color_0, srtb::gui::color_1, srtb::gui::color_overflow,
                                        d_intensity.get(), d_image.get(), nullptr));
    cuda_check(cudaMemcpyAsync(h_image.get(), d_image.get(), n * sizeof(uint32_t), cudaMemcpyDeviceToHost, q.stream()),
               "D2H thumbnail");
    q.wait();  // drop-in contract: the reference's copy ends in .wait()
    return srtb::work::draw_spectrum_work_2{h_image, w.data_stream_id, out_width, out_height};
  }
};

/** <baseband_output_file_prefix>waterfall.<data_stream_id>.ppm: binary P6, RGB (alpha dropped), row 0 = channel 0,
 *  written to a temporary name and renamed over the previous one, so a reader never sees a partial image */
inline bool write_waterfall_ppm(const srtb::work::draw_spectrum_work_2& w) {
  const std::string path =
      srtb::config.baseband_output_file_prefix + "waterfall." + std::to_string(w.data_stream_id) + ".ppm";
  const std::string tmp = path + ".tmp";
  std::vector<unsigned char> rgb(w.width * w.height * 3);
  const uint32_t* px = w.ptr.get();
  for (size_t i = 0; i < w.width * w.height; i++) {
    rgb[3 * i + 0] = static_cast<unsigned char>(px[i] >> 16);
    rgb[3 * i + 1] = static_cast<unsigned char>(px[i] >> 8);
    rgb[3 * i + 2] = static_cast<unsigned char>(px[i]);
  }
  std::ofstream f{tmp, std::ios::binary | std::ios::trunc};
  f << "P6\n" << w.width << " " << w.height << "\n255\n";
  f.write(reinterpret_cast<const char*>(rgb.data()), static_cast<std::streamsize>(rgb.size()));
  f.close();  // a write error may only show when the buffer is flushed here (a full disk)
  std::error_code ec;
  if (!f) {
    SRTB_LOGW << " [waterfall] " << "cannot write " << tmp << "; " << path << " is left as it was";
    std::filesystem::remove(tmp, ec);
    return false;
  }
  std::filesystem::rename(tmp, path, ec);
  if (ec) {
    SRTB_LOGW << " [waterfall] " << "cannot rename " << tmp << " to " << path << ": " << ec.message();
    std::filesystem::remove(tmp, ec);
    return false;
  }
  return true;
}

}  // namespace pipeline
}  // namespace srtb
