// srtb/pipeline/write_signal_pipe.hpp — candidate sink
// (reference: userspace/include/srtb/pipeline/write_signal_pipe.hpp:77-284): a work is kept iff it
// carries at least one time series (file mode), or — in real-time mode (no input_file_path) — also if
// its timestamp lies within 0.45 block lengths of a recent positive (:96-140, so the other
// polarisation / neighbouring blocks of a detection are kept). For a kept work it writes
//   <prefix><counter>.bin            raw baseband block                                (:159-206)
//   <prefix><counter>.<i>.npy        complex64 dynamic spectrum, shape {batch_size, count} (:209-246)
//   <prefix><counter>.<boxcar>.tim   float32 time series per detected boxcar           (:249-280)
// and, for a DM search (dm_list), <prefix><counter>.dm<DM>.<boxcar>.tim and <prefix><counter>.<id>.dm_sweep.csv.
// With dm_search_candidates, also <prefix><counter>.<id>.candidates.csv: the block's single-pulse candidates. With
// signal_detect_candidates the block path writes the same file at its one DM, and <prefix><counter>.sum.candidates.csv
// for the total intensity (signal_detect_sum_polarizations).
// With candidate_cutouts = N, beside each candidate file: <stem>.<id>.cutout_ft.npy and .cutout_dmt.npy (float32
// [N'][nsub][W] and [N'][n_rows][W]) and <stem>.<id>.cutouts.csv, the N' <= N highest-S/N candidates' cut-outs (.sum.
// for the total intensity's file).
// With signal_detect_sum_polarizations, a block whose total intensity is positive keeps every stream's work, and the
// first stream's work writes the sum's series as <prefix><counter>.sum.<boxcar>.tim (once per block).
// counter = udp_packet_counter, or the timestamp when there is none (:145-148).
// Differences: files are written synchronously on the pipe's thread (the reference posts to thread
// pools), and the .npy index is incremented until the name is free (the reference's loop never
// increments `i`, :232-236).
#pragma once
#include <complex>
#include <cstdint>
#include <cstdio>
#include <deque>
#include <filesystem>
#include <fstream>
#include <optional>
#include <stop_token>
#include <string>
#include <vector>

#include "srtb/config.hpp"
#include "srtb/cuda_queue.hpp"
#include "srtb/io/npy.hpp"
#include "srtb/log.hpp"
#include "srtb/work.hpp"

namespace srtb {
namespace pipeline {

class write_signal_pipe {
 protected:
  srtb::cuda_queue q;
  std::deque<uint64_t> recent_positive_timestamps;
  std::deque<srtb::work::write_signal_work> recent_negative_works;
  size_t written_ = 0;

 public:
  explicit write_signal_pipe(srtb::cuda_queue q_) : q{q_} {
    const std::string check = srtb::config.baseband_output_file_prefix + ".check";
    std::ofstream f(check, std::ios::binary);
    if (!f) {
      SRTB_LOGE << " [write_signal_pipe] " << "cannot open file " << check;
      throw std::runtime_error("[write_signal_pipe] cannot open file " + check);
    }
  }
  size_t written() const { return written_; }

  /** the keep/drop decision alone (host logic; testable without a GPU) */
  std::optional<srtb::work::write_signal_work> select(srtb::work::write_signal_work work) {
    std::optional<srtb::work::write_signal_work> keep;
    const bool has_signal = !work.time_series.empty() || work.sum_positive;
    const bool real_time = srtb::config.input_file_path.empty();
    const double window = 0.45 * 1e9 * (double)srtb::config.baseband_input_count / srtb::config.baseband_sample_rate;
    auto near_positive = [&](uint64_t ts) {
      for (auto t : recent_positive_timestamps)
        if (std::abs(static_cast<double>(static_cast<int64_t>(ts - t))) < window) return true;
      return false;
    };
    while (real_time && !recent_positive_timestamps.empty() &&
           static_cast<int64_t>(work.timestamp - recent_positive_timestamps.front()) > 5 * window)
      recent_positive_timestamps.pop_front();
    if (has_signal) {
      recent_positive_timestamps.push_back(work.timestamp);
      keep = std::move(work);
    } else if (real_time) {
      if (near_positive(work.timestamp)) keep = std::move(work);
      else recent_negative_works.push_back(std::move(work));
    }
    if (real_time && !keep && !recent_negative_works.empty()) {
      auto w2 = std::move(recent_negative_works.front());
      recent_negative_works.pop_front();
      if (near_positive(w2.timestamp)) keep = std::move(w2);
    }
    return keep;
  }

  auto operator()(std::stop_token, srtb::work::write_signal_work work) {
    if (auto keep = select(std::move(work))) write(*keep);
    return std::optional{srtb::work::dummy_work{}};
  }

  void write(const srtb::work::write_signal_work& w) {
    uint64_t counter = w.udp_packet_counter;
    if (counter == w.no_udp_packet_counter) counter = w.timestamp;
    const std::string stem = srtb::config.baseband_output_file_prefix + std::to_string(counter);
    SRTB_LOGI << " [write_signal_pipe] " << "Begin writing baseband data, file_counter = " << counter;
    if (w.baseband_data.baseband_ptr) {
      std::ofstream f(stem + ".bin", std::ios::binary | std::ios::trunc);
      f.write(reinterpret_cast<const char*>(w.baseband_data.baseband_ptr.get()),
              (std::streamsize)w.baseband_data.baseband_input_bytes);
    } else {
      SRTB_LOGE << " [write_signal_pipe] " << "baseband pointer not valid!";
    }
    if (w.ptr) {
      const size_t total = w.count * w.batch_size;
      std::vector<std::complex<srtb::real>> h(total);
      cuda_check(cudaSetDevice(q.device()), "cudaSetDevice");
      cuda_check(cudaMemcpyAsync(h.data(), w.ptr.get(), total * sizeof(h[0]), cudaMemcpyDeviceToHost, q.stream()),
                 "D2H spectrum");
      q.wait();
      size_t i = 0;
      std::string path;
      do {
        path = stem + "." + std::to_string(i++) + ".npy";
      } while (std::filesystem::exists(path));
      srtb::io::npy_save(path, h.data(), std::vector<size_t>{w.batch_size, w.count});
    }
    write_series(w, stem);
    written_++;
  }

  /** the host-side files of a kept work: <stem>.<boxcar>.tim per series, <stem>.sum.<boxcar>.tim per positive series of
   *  the total-intensity detector (first stream's work only). A DM search's work (non-empty dm_trials)
   *  names the DM its series belong to, <stem>.dm<DM>.<boxcar>.tim, and also gets <stem>.<data_stream_id>.dm_sweep.csv,
   *  one row per trial and boxcar (one row with zero boxcar fields for a trial whose detector was disabled): the S/N
   *  against DM that tells a dispersed pulse, which peaks at its DM, from RFI, which peaks at DM 0. */
  static void write_series(const srtb::work::write_signal_work& w, const std::string& stem) {
    const bool sweep = !w.dm_trials.empty();
    auto fmt = [](const char* f, double v) {
      char buf[64];
      std::snprintf(buf, sizeof buf, f, v);
      return std::string{buf};
    };
    const std::string dm_part = sweep ? ".dm" + fmt("%g", w.dm) : "";
    for (const auto& ts : w.time_series) {
      std::ofstream f(stem + dm_part + "." + std::to_string(ts.boxcar_length) + ".tim", std::ios::binary | std::ios::trunc);
      f.write(reinterpret_cast<const char*>(ts.h_time_series.get()), (std::streamsize)(ts.time_series_length * sizeof(srtb::real)));
    }
    for (const auto& ts : w.sum_time_series) {
      std::ofstream f(stem + ".sum." + std::to_string(ts.boxcar_length) + ".tim", std::ios::binary | std::ios::trunc);
      f.write(reinterpret_cast<const char*>(ts.h_time_series.get()), (std::streamsize)(ts.time_series_length * sizeof(srtb::real)));
    }
    if (!sweep) {
      // signal_detect_candidates: the block path's candidates, and the total intensity's on the first stream's work
      if (w.has_candidates) write_candidates(w, stem);
      if (w.has_sum_candidates) write_candidate_rows(w, w.sum_candidates, stem + ".sum.candidates.csv");
      if (w.sum_cutouts) write_cutouts(w, *w.sum_cutouts, stem + ".sum");
      return;
    }
    std::ofstream f(stem + "." + std::to_string(w.data_stream_id) + ".dm_sweep.csv", std::ios::trunc);
    f << "dm,detect_enabled,boxcar_length,series_length,signal_count,threshold,peak_snr,peak_index\n";
    for (const auto& t : w.dm_trials) {
      const std::string head = fmt("%g", t.dm) + "," + (t.detect_enabled ? "1" : "0") + ",";
      if (t.boxcars.empty()) f << head << "0,0,0,0,0,0\n";
      for (const auto& b : t.boxcars)
        f << head << b.boxcar_length << "," << b.series_length << "," << b.signal_count << ","
          << fmt("%.9g", b.threshold) << "," << fmt("%.9g", b.peak_snr) << "," << b.peak_index << "\n";
    }
    if (!f) SRTB_LOGE << " [write_signal_pipe] " << "cannot write " << stem << ".dm_sweep.csv";
    if (w.has_candidates) write_candidates(w, stem);
  }

  /** <stem>.<data_stream_id>.candidates.csv: a header row, then one row per candidate in the block's own share, those
   *  whose window is below the work's candidate_share (candidate_share() in baseband_chain_pipe.hpp). sample = window +
   *  the work's offset (S- for the incoherent search), time = (first_sample + 2C sample) / sample_rate in seconds from
   *  input_file_offset_bytes, topocentric and referred to f_c (empty without a first_sample). The block path
   *  (signal_detect_candidates) writes the same columns: dm = dm_low = dm_high = the block's dm, trial 0. */
  static void write_candidates(const srtb::work::write_signal_work& w, const std::string& stem) {
    write_candidate_rows(w, w.candidates, stem + "." + std::to_string(w.data_stream_id) + ".candidates.csv");
    if (w.cutouts) write_cutouts(w, *w.cutouts, stem + "." + std::to_string(w.data_stream_id));
  }

  /** candidate_cutouts: <base>.cutout_ft.npy, <base>.cutout_dmt.npy and <base>.cutouts.csv, a header row, then one row
   *  per cut-out: its row in the candidate file, center (spectrum sample at bin W/2), decimation, the time of bin 0
   *  (spectrum sample center - (W/2) decimation, as candidates.csv defines time; empty without a first_sample) and the
   *  DMs of the plane's first and last rows */
  static void write_cutouts(const srtb::work::write_signal_work& w, const srtb::work::cutout_set& c,
                            const std::string& base) {
    const size_t n = c.rows.size();
    srtb::io::npy_save(base + ".cutout_ft.npy", c.ft.data(), std::vector<size_t>{n, c.nsub, c.width});
    srtb::io::npy_save(base + ".cutout_dmt.npy", c.dmt.data(), std::vector<size_t>{n, c.n_rows, c.width});
    auto fmt = [](const char* f, double v) {
      char buf[64];
      std::snprintf(buf, sizeof buf, f, v);
      return std::string{buf};
    };
    const uint64_t two_c = 2 * (uint64_t)w.batch_size;
    const bool placed = w.first_sample != w.no_first_sample;
    std::ofstream f(base + ".cutouts.csv", std::ios::trunc);
    f << "candidate,center,decimation,time,dm_row_low,dm_row_high\n";
    for (const auto& r : c.rows) {
      const double bin0 = (double)r.center - (double)(c.width / 2) * (double)r.decimation;
      const std::string time =
          placed ? fmt("%.12g", ((double)w.first_sample + (double)two_c * bin0) / srtb::config.baseband_sample_rate) : "";
      f << r.candidate << "," << r.center << "," << r.decimation << "," << time << "," << fmt("%.9g", r.dm_row_low)
        << "," << fmt("%.9g", r.dm_row_high) << "\n";
    }
    if (!f) SRTB_LOGE << " [write_signal_pipe] " << "cannot write " << base << ".cutouts.csv";
  }

  /** write_candidates' file of `candidates` at `path`, under w's share, offset, geometry and first sample */
  static void write_candidate_rows(const srtb::work::write_signal_work& w,
                                   const std::vector<srtb::work::dm_candidate>& candidates, const std::string& path) {
    auto fmt = [](const char* f, double v) {
      char buf[64];
      std::snprintf(buf, sizeof buf, f, v);
      return std::string{buf};
    };
    const uint64_t two_c = 2 * (uint64_t)w.batch_size;
    const bool placed = w.first_sample != w.no_first_sample;
    std::ofstream f(path, std::ios::trunc);
    f << "snr,dm,boxcar_length,sample,time,members,dm_low,dm_high,span_begin,span_end,trial,peak_index\n";
    for (const auto& c : candidates) {
      if (c.window >= w.candidate_share) continue;
      const uint64_t sample = c.window + w.candidate_sample_offset;
      const std::string time =
          placed ? fmt("%.12g", ((double)w.first_sample + (double)two_c * (double)sample) / srtb::config.baseband_sample_rate)
                 : "";
      f << fmt("%.9g", c.snr) << "," << fmt("%g", c.dm) << "," << c.boxcar_length << "," << sample << "," << time << ","
        << c.members << "," << fmt("%g", c.dm_low) << "," << fmt("%g", c.dm_high) << "," << c.span_begin << ","
        << c.span_end << "," << c.trial << "," << c.peak_index << "\n";
    }
    if (!f) SRTB_LOGE << " [write_signal_pipe] " << "cannot write " << path;
  }
};

}  // namespace pipeline
}  // namespace srtb
