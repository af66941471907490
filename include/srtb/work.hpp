// srtb/work.hpp — work items and work queues of the pipeline, same fields and names as the
// reference (userspace/include/srtb/work.hpp:30-72 work_queue, :102-157 work<T>, :162-285 typedefs).
// Boost.Lockfree / moodycamel are not used: a bounded ring (SPSC use) and a mutex deque (MPMC use)
// provide the same push / pop / read_available / empty surface.
#pragma once
#include <array>
#include <atomic>
#include <cstddef>
#include <cstdint>
#include <deque>
#include <memory>
#include <mutex>
#include <vector>

#include "srtb/config.hpp"

namespace srtb {

/** bounded single-producer single-consumer ring, capacity fixed at compile time */
template <typename T, size_t capacity>
class spsc_ring {
  std::array<T, capacity + 1> slots_{};
  std::atomic<size_t> head_{0}, tail_{0};  // head: next pop, tail: next push

 public:
  bool push(const T& v) {
    const size_t t = tail_.load(std::memory_order_relaxed);
    const size_t next = (t + 1) % (capacity + 1);
    if (next == head_.load(std::memory_order_acquire)) return false;  // full
    slots_[t] = v;
    tail_.store(next, std::memory_order_release);
    return true;
  }
  bool pop(T& out) {
    const size_t h = head_.load(std::memory_order_relaxed);
    if (h == tail_.load(std::memory_order_acquire)) return false;  // empty
    out = std::move(slots_[h]);
    slots_[h] = T{};
    head_.store((h + 1) % (capacity + 1), std::memory_order_release);
    return true;
  }
  size_t read_available() const {
    const size_t h = head_.load(std::memory_order_acquire), t = tail_.load(std::memory_order_acquire);
    return (t + capacity + 1 - h) % (capacity + 1);
  }
  bool empty() const { return read_available() == 0; }
};

/** unbounded multi-producer multi-consumer queue */
template <typename T>
class mpmc_queue {
  mutable std::mutex m_;
  std::deque<T> q_;

 public:
  bool push(const T& v) {
    std::lock_guard<std::mutex> g{m_};
    q_.push_back(v);
    return true;
  }
  bool pop(T& out) {
    std::lock_guard<std::mutex> g{m_};
    if (q_.empty()) return false;
    out = std::move(q_.front());
    q_.pop_front();
    return true;
  }
  size_t read_available() const {
    std::lock_guard<std::mutex> g{m_};
    return q_.size();
  }
  bool empty() const { return read_available() == 0; }
};

/** multi-producer multi-consumer queue holding at most `capacity` works: push fails (returns false) when it is full,
 *  so a loose out-functor drops the work instead of queueing it */
template <typename T>
class bounded_mpmc_queue {
  mutable std::mutex m_;
  std::deque<T> q_;
  size_t capacity_;

 public:
  using work_type = T;
  explicit bounded_mpmc_queue(size_t capacity = srtb::work_queue_capacity) : capacity_{capacity} {}
  bool push(const T& v) {
    std::lock_guard<std::mutex> g{m_};
    if (q_.size() >= capacity_) return false;
    q_.push_back(v);
    return true;
  }
  bool pop(T& out) {
    std::lock_guard<std::mutex> g{m_};
    if (q_.empty()) return false;
    out = std::move(q_.front());
    q_.pop_front();
    return true;
  }
  size_t read_available() const {
    std::lock_guard<std::mutex> g{m_};
    return q_.size();
  }
  bool empty() const { return read_available() == 0; }
};

// work_queue<T, spsc, fixed_size, capacity> as in the reference; spsc = false -> MPMC
template <typename T, bool spsc = true, bool fixed_size = srtb::work_queue_fixed_size,
          size_t capacity = srtb::work_queue_capacity>
class work_queue : public spsc_ring<T, capacity> {
 public:
  using work_type = T;
};
template <typename T, bool fixed_size, size_t capacity>
class work_queue<T, false, fixed_size, capacity> : public mpmc_queue<T> {
 public:
  using work_type = T;
};

namespace pipeline {
struct dummy_work {};  // pipeline/framework/dummy_pipe.hpp
}  // namespace pipeline

namespace work {

using dummy_work = srtb::pipeline::dummy_work;

/** original baseband of a block, kept so a positive detection can be written out (work.hpp:88-96) */
struct baseband_data_holder {
  std::shared_ptr<std::byte> baseband_ptr;
  size_t baseband_input_bytes = 0;
};

template <typename T>
struct work {
  T ptr{};
  size_t count = 0;       // shape[0]
  size_t batch_size = 1;  // shape[1]
  uint64_t timestamp = 0;
  uint64_t udp_packet_counter = static_cast<uint64_t>(-1);
  uint32_t data_stream_id = 0;
  static constexpr uint64_t no_udp_packet_counter = static_cast<uint64_t>(-1);
  // the block's place in a recording, in baseband samples per stream (read_file_pipe): its first sample, counted from
  // input_file_offset_bytes, and the samples actually read (the rest of the block is zero fill). Blocks from other
  // sources keep no_first_sample and are never folded
  static constexpr uint64_t no_first_sample = static_cast<uint64_t>(-1);
  uint64_t first_sample = no_first_sample;
  uint64_t valid_samples = 0;
  baseband_data_holder baseband_data;

  template <typename U>
  void move_parameter_from(work<U>&& other) {
    timestamp = other.timestamp;
    udp_packet_counter = other.udp_packet_counter;
    data_stream_id = other.data_stream_id;
    first_sample = other.first_sample;
    valid_samples = other.valid_samples;
    baseband_data = std::move(other.baseband_data);
  }
  template <typename U>
  void copy_parameter_from(const work<U>& other) {
    timestamp = other.timestamp;
    udp_packet_counter = other.udp_packet_counter;
    data_stream_id = other.data_stream_id;
    first_sample = other.first_sample;
    valid_samples = other.valid_samples;
    baseband_data = other.baseband_data;
  }
};

using complex_ptr = std::shared_ptr<srtb::complex<srtb::real>>;
using copy_to_device_work = work<std::shared_ptr<std::byte>>;
using unpack_work = work<std::shared_ptr<std::byte>>;
using fft_1d_r2c_work = work<std::shared_ptr<srtb::real>>;
using fft_1d_c2c_work = work<complex_ptr>;
using rfi_mitigation_s1_work = work<complex_ptr>;
using dedisperse_work = work<complex_ptr>;
using ifft_1d_c2c_work = work<complex_ptr>;
using refft_1d_c2c_work = work<complex_ptr>;
using watfft_1d_c2c_work = work<complex_ptr>;
using rfi_mitigation_s2_work = work<complex_ptr>;
using signal_detect_work = work<complex_ptr>;
using write_file_work = work<complex_ptr>;

/** one detected time series: host copy + boxcar length (work.hpp:240-247; no transfer_event —
 *  the copy has completed when the detect pipe returns) */
struct time_series_holder {
  std::shared_ptr<srtb::real> h_time_series;
  size_t time_series_length = 0;
  size_t boxcar_length = 0;
  size_t signal_count = 0;
};

/** one trial of a DM search on one data stream: its DM, whether the detector ran, and per boxcar what it found */
struct dm_trial_summary {
  struct boxcar {
    size_t boxcar_length = 0;
    size_t series_length = 0;
    size_t signal_count = 0;
    float threshold = 0;
    float peak_snr = 0;     // largest series value / sqrt(variance)
    size_t peak_index = 0;  // first index of that value in the series
  };
  srtb::real dm = 0;
  bool detect_enabled = false;
  std::vector<boxcar> boxcars;
};

/** one block folded at fold_period: where it lies in the recording and what srtb_b200_fold (and, with fold_coherence,
 *  srtb_b200_fold_coherence) returned for it */
struct fold_block {
  uint64_t block_index = 0;   // first_sample / (N - R): blocks tile the recording in steps of N - R samples
  uint64_t first_sample = 0;
  size_t streams = 0, subbands = 0, bins = 0;
  std::vector<double> profile;  // [streams][subbands][bins]
  std::vector<uint64_t> hits;   // [bins]
  std::vector<uint32_t> kept;   // [streams][subbands]
  // fold_coherence only (srtb_b200_fold_coherence of streams 0 and 1; empty otherwise): AA, BB, CR, CI and the
  // channels kept in both streams
  std::vector<double> coherence;         // [4][subbands][bins]
  std::vector<uint32_t> coherence_kept;  // [subbands]
};

/** one single-pulse candidate of a DM search (srtb_b200_candidate): its representative event's S/N, DM, boxcar, trial
 *  and window (the series index its boxcar window starts at), and the members' count, DM range and span */
struct dm_candidate {
  float snr = 0, dm = 0, dm_low = 0, dm_high = 0;
  uint64_t boxcar_length = 0, peak_index = 0, window = 0, members = 0, span_begin = 0, span_end = 0;
  uint32_t trial = 0;
};

/** candidate_cutouts: the cut-outs of one candidate file (srtb_b200_candidate_cutouts), in S/N order, highest first */
struct cutout_set {
  size_t width = 0, nsub = 0, n_rows = 0;
  std::vector<float> ft;   // [n][nsub][width]
  std::vector<float> dmt;  // [n][n_rows][width]
  struct row {
    uint64_t candidate = 0;  // 0-based row in the candidate file
    int64_t center = 0;      // spectrum sample at bin width/2
    uint32_t decimation = 0;
    float dm_row_low = 0, dm_row_high = 0;  // the plane's first and last rows' DMs
  };
  std::vector<row> rows;
};

struct write_signal_work : public write_file_work {
  std::vector<time_series_holder> time_series;  // non-empty <=> has_signal
  size_t zero_count = 0;
  // signal_detect_sum_polarizations: every stream's work of a block whose total-intensity detector is positive has
  // sum_positive set (the sink keeps it); the block's first stream also carries that detector's result
  bool sum_positive = false;
  bool carries_sum = false;
  size_t sum_zero_count = 0;
  std::vector<size_t> sum_signal_count;               // per boxcar
  std::vector<time_series_holder> sum_time_series;    // its positive series
  // DM search only (dm_sweep_chain_pipe): the best trial's DM, which ptr and time_series belong to, and every trial
  srtb::real dm = 0;
  std::vector<dm_trial_summary> dm_trials;
  // dm_search_candidates: the block's candidates, the bound on their window of the block's own share (write_signal_pipe
  // writes those below it) and the spectrum sample of series index 0 (S- for the incoherent search, 0 for the sweep)
  bool has_candidates = false;
  std::vector<dm_candidate> candidates;
  uint64_t candidate_share = 0;
  uint64_t candidate_sample_offset = 0;
  // signal_detect_candidates with the total-intensity sum: the sum's candidates, on the first stream's work (same share)
  bool has_sum_candidates = false;
  std::vector<dm_candidate> sum_candidates;
  // candidate_cutouts: the cut-outs of candidates' and of sum_candidates' files (null when off or empty)
  std::shared_ptr<const cutout_set> cutouts, sum_cutouts;
  // fold_period: the block's fold (srtb_b200_fold), carried by the block's first stream
  std::shared_ptr<const fold_block> fold;
};

/** a [batch_size][count] complex dynamic spectrum on the device, to be turned into a waterfall thumbnail
 *  (work.hpp:267-271); a write_signal_work converts to it */
using simplify_spectrum_work = work<complex_ptr>;

/** ARGB32 thumbnail of width * height pixels in host memory, row 0 = channel 0 (work.hpp:276-284) */
struct draw_spectrum_work_2 {
  std::shared_ptr<uint32_t> ptr;
  uint32_t data_stream_id = 0;
  size_t width = 0;
  size_t height = 0;
};

}  // namespace work
}  // namespace srtb
