// src/main.cpp — `srtb_b200`, the drop-in executable for the baseband -> single-pulse path.
// Equivalent of the reference's main (/root/reference/userspace/src/main.cpp:88-328) for the part of it that is
// in scope (SURVEY §8): same config surface (srtb_config.cfg / --key value, expressions and all), same source
// selection (input_file_path -> read_file_pipe, else one UDP receiver per address/port, main.cpp:125-168), same sink
// selection (baseband_write_all -> write_file_pipe, else write_signal_pipe, main.cpp:206-216). Between source and
// sink the seven device pipes run as the fused chain pipe (baseband_chain_pipe = srtb_b200_submit_block_ex /
// collect_block_ex), several per GPU, and — new with respect to the reference, which drives one device
// (main.cpp:99) — blocks are dealt round-robin over every visible GPU (block k -> GPU k mod G, SURVEY §8e; no
// collective on the data path). With gui_enable, the chain's spectra also feed a loose side branch per GPU
// (main.cpp:197-201,220-228): simplify_spectrum_pipe_2 on that GPU makes the waterfall thumbnail and one sink writes it
// to <baseband_output_file_prefix>waterfall.<data_stream_id>.ppm, replaced on every block (the headless counterpart of
// the reference's refreshed window). The Qt window itself and the termination handler are out of scope.
//
// Extra options (not part of srtb::configs; consumed here before the reference-style parser sees argv):
//   --gpu_devices 0,1,...   GPUs to use (default: all visible)      --chains_per_gpu N   chain pipes per GPU (default 2)
//   --ring_depth N          blocks in flight per chain pipe (1..3, default 3)
//   --synthetic_udp_rate R  no socket: a synthetic packet stream (the format's framing, Gaussian 8-bit noise) released at
//                           R samples/s per receiver like a NIC would (0 = as fast as it is taken); with
//   --synthetic_duration S  seconds of stream (default 10); prints one JSON line with blocks, rate and lost packets
//   --discard_output 1      count results instead of writing candidate files
// With dm_list set (a srtb::configs key: --dm_list "0:100:5" or a .cfg line), every block is searched over those trial
// DMs by dm_sweep_chain_pipe instead of baseband_chain_pipe at `dm` (which is then not used); its pipes run without a
// ring, so --ring_depth is ignored. The sink then writes the best trial's files and a per-stream S/N-versus-DM table.
// With incoherent_dm_list set instead (--incoherent_dm_list, same syntax), baseband_chain_pipe dedisperses coherently at
// `dm` and then searches those trial DMs incoherently on each stream's dynamic spectrum; the ring is kept and the sink
// writes the same files for the best incoherent trial.
// With fold_period set (a recording only), every block is also folded at that period on the device after its
// detector, and the sink adds the folds into subintegrations: <prefix>fold.npy, fold.weights.npy and fold.json. With
// fold_coherence also the coherence products of streams 0 and 1: fold.coherence.npy and fold.coherence.weights.npy.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <csignal>
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <thread>
#include <vector>

#include "srtb/config.hpp"
#include "srtb/cuda_queue.hpp"
#include "srtb/io/udp_block_assembler.hpp"
#include "srtb/memory.hpp"
#include "srtb/pipeline/baseband_chain_pipe.hpp"
#include "srtb/pipeline/dm_sweep_chain_pipe.hpp"
#include "srtb/pipeline/fold_pipe.hpp"
#include "srtb/pipeline/framework/pipe.hpp"
#include "srtb/pipeline/framework/pipe_io.hpp"
#include "srtb/pipeline/read_file_pipe.hpp"
#include "srtb/pipeline/spectrum_pipe.hpp"
#include "srtb/pipeline/udp_receiver_pipe.hpp"
#include "srtb/pipeline/write_file_pipe.hpp"
#include "srtb/pipeline/write_signal_pipe.hpp"
#include "srtb/program_options.hpp"
#include "srtb/work.hpp"

namespace {

std::atomic<bool> g_interrupted{false};
void on_signal(int) { g_interrupted = true; }

using copy_queue = srtb::work_queue<srtb::work::copy_to_device_work, false>;
using output_queue = srtb::work_queue<srtb::work::write_signal_work, false>;
using draw_queue = srtb::bounded_mpmc_queue<srtb::work::draw_spectrum_work_2>;

/** writes each thumbnail as the stream's PPM; `written` counts them */
struct waterfall_sink {
  std::shared_ptr<std::atomic<uint64_t>> written;
  std::optional<srtb::work::dummy_work> operator()(std::stop_token, srtb::work::draw_spectrum_work_2 w) {
    srtb::pipeline::write_waterfall_ppm(w);
    (*written)++;
    return srtb::work::dummy_work{};
  }
};

/** source -> per-GPU queues: block k goes to GPU k mod G (all streams of a block stay together) */
struct round_robin_out_functor {
  std::vector<std::shared_ptr<copy_queue>> queues;
  std::shared_ptr<std::atomic<uint64_t>> submitted;
  std::shared_ptr<std::atomic<int64_t>> first_ns = std::make_shared<std::atomic<int64_t>>(0);  // first block handed over
  void operator()(std::stop_token st, srtb::work::copy_to_device_work w) {
    if (submitted->load() == 0)
      first_ns->store(std::chrono::duration_cast<std::chrono::nanoseconds>(
                          std::chrono::steady_clock::now().time_since_epoch()).count());
    auto& q = queues[submitted->load() % queues.size()];
    while (!q->push(w)) {
      if (st.stop_requested()) return;
      std::this_thread::sleep_for(std::chrono::microseconds(50));
    }
    (*submitted)++;
  }
};

/** sink wrapper: counts finished works so file replays know when everything has drained */
// signal_detect_sum_polarizations: one line per block with the total-intensity detector's counts
void log_sum(const srtb::work::write_signal_work& w) {
  if (!w.carries_sum) return;
  std::string counts;
  for (size_t c : w.sum_signal_count) counts += (counts.empty() ? "" : ",") + std::to_string(c);
  SRTB_LOGI << " [main] " << "block " << w.timestamp << ": total intensity " << (w.sum_positive ? "positive" : "negative")
            << ", masked channels " << w.sum_zero_count << ", signal counts per boxcar [" << counts << "]";
}

// fold_period: the block's fold goes to the accumulator (null when folding is off)
void add_fold(const std::shared_ptr<srtb::pipeline::fold_accumulator>& folds, const srtb::work::write_signal_work& w) {
  if (folds && w.fold) folds->add(w.fold);
}

template <typename Sink>
struct counting_sink {
  std::shared_ptr<Sink> sink;
  std::shared_ptr<std::atomic<uint64_t>> done;
  std::shared_ptr<srtb::pipeline::fold_accumulator> folds;
  std::optional<srtb::work::dummy_work> operator()(std::stop_token st, srtb::work::write_signal_work w) {
    log_sum(w);
    add_fold(folds, w);
    (*sink)(st, std::move(w));
    (*done)++;
    return srtb::work::dummy_work{};
  }
};

std::string take_option(std::vector<std::string>& args, const std::string& name, const std::string& def) {
  for (size_t i = 0; i < args.size(); i++) {
    if (args[i] == "--" + name && i + 1 < args.size()) {
      std::string v = args[i + 1];
      args.erase(args.begin() + (long)i, args.begin() + (long)i + 2);
      return v;
    }
    if (args[i].rfind("--" + name + "=", 0) == 0) {
      std::string v = args[i].substr(name.size() + 3);
      args.erase(args.begin() + (long)i);
      return v;
    }
  }
  return def;
}

/** results counted, nothing written (throughput runs) */
struct discard_sink {
  std::shared_ptr<std::atomic<uint64_t>> done, positives;
  std::shared_ptr<srtb::pipeline::fold_accumulator> folds;
  std::optional<srtb::work::dummy_work> operator()(std::stop_token, srtb::work::write_signal_work w) {
    log_sum(w);
    add_fold(folds, w);
    if (!w.time_series.empty()) (*positives)++;
    (*done)++;
    return srtb::work::dummy_work{};
  }
};

struct synthetic_stats {
  std::shared_ptr<std::atomic<uint64_t>> received = std::make_shared<std::atomic<uint64_t>>(0);
  std::shared_ptr<std::atomic<uint64_t>> lost = std::make_shared<std::atomic<uint64_t>>(0);
};

/** udp_receiver_pipe over the paced synthetic provider; publishes its packet statistics when the stream ends */
template <typename Backend>
struct synthetic_receiver_pipe {
  using provider = srtb::io::udp::paced_packet_provider<Backend>;
  srtb::pipeline::udp_receiver_pipe<provider, Backend> inner;
  synthetic_stats stats;
  synthetic_receiver_pipe(provider p, size_t id, synthetic_stats st) : inner{std::move(p), id}, stats{st} {}
  std::optional<srtb::work::copy_to_device_work> operator()(std::stop_token st, srtb::work::dummy_work d) {
    auto w = inner(st, d);
    stats.received->store(inner.received_packets());
    stats.lost->store(inner.lost_packets());
    return w;
  }
};

template <typename Backend>
std::jthread start_synthetic_source(size_t id, double samples_per_s, double seconds, round_robin_out_functor out,
                                    synthetic_stats stats) {
  using namespace srtb::pipeline;
  // four distinct blocks of Gaussian-ish 8-bit noise (sum of four uniform bytes, sigma ~ 20 counts), framed and replayed
  const size_t block_bytes = srtb::config.baseband_input_count * Backend::data_stream_count;
  std::vector<std::byte> payload(4 * block_bytes);
  uint64_t x = 0x9E3779B97F4A7C15ull + id;
  for (size_t i = 0; i < payload.size(); i++) {
    x ^= x << 13;
    x ^= x >> 7;
    x ^= x << 17;
    const int sum = (int)(x & 0xff) + (int)((x >> 8) & 0xff) + (int)((x >> 16) & 0xff) + (int)((x >> 24) & 0xff) - 510;
    payload[i] = static_cast<std::byte>(static_cast<int8_t>(sum * 20 / 148));
  }
  typename synthetic_receiver_pipe<Backend>::provider prov{payload, samples_per_s * (double)Backend::data_stream_count,
                                                            (uint64_t)id << 40};
  prov.run_for(seconds);
  return start_pipe<synthetic_receiver_pipe<Backend>>(dummy_in_functor<>{}, out, std::move(prov), id, stats);
}

template <typename Backend>
std::jthread start_udp_source(size_t id, const std::string& address, unsigned short port, round_robin_out_functor out) {
  using namespace srtb::pipeline;
  using provider = srtb::io::udp::recvfrom_packet_provider;
  return start_pipe<udp_receiver_pipe<provider, Backend>>(dummy_in_functor<>{}, out, provider{address, port}, id);
}

}  // namespace

int main(int argc, char** argv) {
  using namespace srtb::pipeline;
  // separate hardware work queues for the streams of a context's two lanes (see INTEGRATION.md): the documented default,
  // pinned before CUDA initialises; an exported value wins
  setenv("CUDA_DEVICE_MAX_CONNECTIONS", "8", /*overwrite=*/0);
  std::vector<std::string> args(argv + 1, argv + argc);
  const std::string devices_opt = take_option(args, "gpu_devices", "");
  const int chains_per_gpu = std::max(1, std::atoi(take_option(args, "chains_per_gpu", "2").c_str()));
  const int ring_depth = std::max(1, std::atoi(take_option(args, "ring_depth", "3").c_str()));
  const std::string synth_rate_opt = take_option(args, "synthetic_udp_rate", "");
  const double synth_seconds = std::atof(take_option(args, "synthetic_duration", "10").c_str());
  const bool discard = std::atoi(take_option(args, "discard_output", "0").c_str()) != 0;
  std::vector<char*> av{argv[0]};
  for (auto& a : args) av.push_back(a.data());
  auto& cfg = srtb::config;
  try {
    srtb::program_options::apply_changed_configs(
        srtb::program_options::parse_arguments((int)av.size(), av.data(), cfg.config_file_name), cfg);
  } catch (const std::exception& e) {
    std::fprintf(stderr, "srtb_b200: %s\n", e.what());
    return 2;
  }
  if (cfg.gui_enable && (cfg.gui_pixmap_width == 0 || cfg.gui_pixmap_height == 0)) {
    std::fprintf(stderr, "srtb_b200: gui_enable needs a non-zero gui_pixmap_width and gui_pixmap_height (got %zu x %zu)\n",
                 (size_t)cfg.gui_pixmap_width, (size_t)cfg.gui_pixmap_height);
    return 2;
  }
  try {
    srtb::program_options::check_sum_polarizations(
        cfg, srtb::io::backend_registry::get_data_stream_count(cfg.baseband_format_type));
    srtb::program_options::check_fold(cfg);
    srtb::program_options::check_dm_search_candidates(cfg);
    srtb::program_options::check_signal_detect_candidates(cfg);
    srtb::program_options::check_candidate_cutouts(cfg);
  } catch (const std::exception& e) {
    std::fprintf(stderr, "srtb_b200: %s\n", e.what());
    return 2;
  }

  std::vector<int> devices;
  if (devices_opt.empty()) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
      std::fprintf(stderr, "srtb_b200: no CUDA device (there is no CPU fallback)\n");
      return 3;
    }
    for (int i = 0; i < n; i++) devices.push_back(i);
  } else {
    for (const auto& s : srtb::program_options::split_list(devices_opt, ',')) devices.push_back(std::atoi(s.c_str()));
  }
  const std::vector<srtb::real> dm_trials = srtb::program_options::parse_dm_list(cfg.dm_list);
  const bool dm_sweep = !dm_trials.empty();
  if (dm_sweep) {
    SRTB_LOGI << " [main] " << "DM search: " << dm_trials.size() << " trial DM(s) from "
              << *std::min_element(dm_trials.begin(), dm_trials.end()) << " to "
              << *std::max_element(dm_trials.begin(), dm_trials.end()) << "; dm = " << cfg.dm << " is not used";
    SRTB_LOGI << " [main] " << devices.size() << " GPU(s), " << chains_per_gpu
              << " DM-sweep pipe(s) each; --ring_depth is ignored (no ring in a DM sweep)";
  } else {
    SRTB_LOGI << " [main] " << devices.size() << " GPU(s), " << chains_per_gpu << " chain pipe(s) each, ring depth "
              << ring_depth;
  }
  const std::vector<srtb::real> inc_trials = srtb::program_options::parse_dm_list(cfg.incoherent_dm_list);
  if (!inc_trials.empty()) {
    uint64_t s_plus = 0, s_minus = 0;
    const size_t C = std::min<size_t>(cfg.spectrum_channel_count, cfg.baseband_input_count / 2);
    if (srtb_b200_incoherent_shifts(C, cfg.baseband_freq_low, cfg.baseband_bandwidth, cfg.baseband_sample_rate, cfg.dm,
                                    inc_trials.data(), inc_trials.size(), nullptr, &s_plus, &s_minus) != 0) {
      std::fprintf(stderr, "srtb_b200: incoherent_dm_list: %s\n", srtb_b200_last_error(nullptr));
      return 2;
    }
    const size_t overlap = srtb::codd::nsamps_reserved_max();
    if (overlap >= cfg.baseband_input_count) {
      std::fprintf(stderr,
                   "srtb_b200: incoherent_dm_list needs a block overlap of %zu samples (S+ = %llu, S- = %llu spectrum "
                   "samples), not less than baseband_input_count = %zu: narrow the trial DMs or enlarge the block\n",
                   overlap, (unsigned long long)s_plus, (unsigned long long)s_minus, (size_t)cfg.baseband_input_count);
      return 2;
    }
    SRTB_LOGI << " [main] " << "incoherent DM search around dm = " << cfg.dm << ": " << inc_trials.size()
              << " incoherent trial DM(s) from " << *std::min_element(inc_trials.begin(), inc_trials.end()) << " to "
              << *std::max_element(inc_trials.begin(), inc_trials.end()) << ", S+ = " << s_plus << ", S- = " << s_minus
              << " spectrum samples, block overlap " << overlap << " samples";
  }
  std::shared_ptr<fold_accumulator> folds;
  if (cfg.fold_period != 0) {
    const fold_parameters fp = fold_parameters::from_config(
        srtb::io::backend_registry::get_data_stream_count(cfg.baseband_format_type), fold_block_step());
    folds = std::make_shared<fold_accumulator>(fp);
    SRTB_LOGI << " [main] " << "folding at P = " << fp.period << " s, Pdot = " << fp.period_derivative << ": "
              << fp.bins << " bin(s), " << fp.subbands << " subband(s) of " << fp.channels / fp.subbands
              << " channel(s), dt = " << fp.dt() << " s, " << fp.block_step / (2 * fp.channels)
              << " spectrum samples per block, " << (fp.subintegration_blocks ? std::to_string(fp.subintegration_blocks)
                                                                              : std::string{"all"})
              << " block(s) per subintegration" << (fp.coherence ? ", with the coherence products of streams 0 and 1" : "");
  }
  // the device chain between source and sink: one DM, or the trial DMs of dm_list
  auto start_chain = [&](auto in, auto out, int dev) {
    if (dm_sweep) return start_pipe<dm_sweep_chain_pipe>(in, out, srtb::cuda_queue{dev});
    return start_pipe<baseband_chain_pipe>(in, out, srtb::cuda_queue{dev}, false, ring_depth);
  };
  const int blocks_in_flight = dm_sweep ? 1 : ring_depth;

  auto submitted = std::make_shared<std::atomic<uint64_t>>(0);
  auto done = std::make_shared<std::atomic<uint64_t>>(0);
  auto out_q = std::make_shared<output_queue>();
  std::vector<std::shared_ptr<copy_queue>> gpu_queues;
  std::vector<std::jthread> threads;

  auto thumbnails_open = std::make_shared<std::atomic<bool>>(false);
  auto thumbnails_accepted = std::make_shared<std::atomic<uint64_t>>(0);
  auto thumbnails_written = std::make_shared<std::atomic<uint64_t>>(0);
  auto thumbnails_dropped = std::make_shared<std::atomic<uint64_t>>(0);
  // the sink's queue is bounded too: a thumbnail pipe waits for room, its own input queue fills, and then the side
  // branch drops blocks, so a slow disk never holds more than a few images and spectra per GPU
  auto draw_q = std::make_shared<draw_queue>(srtb::work_queue_capacity * devices.size());

  // device side: the fused chain, `chains_per_gpu` pipes per GPU on their own CUDA stream / context each
  for (int dev : devices) {
    gpu_queues.push_back(std::make_shared<copy_queue>());
    if (cfg.gui_enable) {
      // the thumbnail side branch is offered each work before the sink's queue, so once the sink has seen a block
      // that block's side-branch decision has been made
      auto thumb_q = std::make_shared<thumbnail_out_functor::queue>(srtb::work_queue_capacity);
      for (int c = 0; c < chains_per_gpu; c++)
        threads.push_back(start_chain(
            idle_queue_in_functor{gpu_queues.back()},
            multiple_works_out_functor{multiple_out_functors_functor{
                thumbnail_out_functor{thumb_q, thumbnails_open, thumbnails_accepted, thumbnails_dropped}, queue_out_functor{out_q}}},
            dev));
      threads.push_back(start_pipe<simplify_spectrum_pipe_2>(queue_in_functor{thumb_q}, queue_out_functor{draw_q},
                                                             srtb::cuda_queue{dev}));
    } else {
      for (int c = 0; c < chains_per_gpu; c++)
        threads.push_back(start_chain(idle_queue_in_functor{gpu_queues.back()},
                                      multiple_works_out_functor{queue_out_functor{out_q}}, dev));
    }
  }
  if (cfg.gui_enable)
    threads.push_back(start_pipe<waterfall_sink>(queue_in_functor{draw_q}, dummy_out_functor<>{}, thumbnails_written));
  // sink (main.cpp:206-216)
  srtb::cuda_queue q0{devices.front()};
  auto positives = std::make_shared<std::atomic<uint64_t>>(0);
  if (discard) {
    threads.push_back(start_pipe<discard_sink>(queue_in_functor{out_q}, dummy_out_functor<>{}, done, positives, folds));
  } else if (cfg.baseband_write_all) {
    SRTB_LOGW << " [main] " << "Writing all baseband data, take care of disk space!";
    threads.push_back(start_pipe<counting_sink<write_file_pipe>>(
        queue_in_functor{out_q}, dummy_out_functor<>{}, std::make_shared<write_file_pipe>(q0), done, folds));
  } else {
    threads.push_back(start_pipe<counting_sink<write_signal_pipe>>(
        queue_in_functor{out_q}, dummy_out_functor<>{}, std::make_shared<write_signal_pipe>(q0), done, folds));
  }
  // source (main.cpp:125-168)
  std::signal(SIGINT, on_signal);
  std::signal(SIGTERM, on_signal);
  round_robin_out_functor rr{gpu_queues, submitted};
  const size_t streams = srtb::io::backend_registry::get_data_stream_count(cfg.baseband_format_type);
  // a live stream cannot wait for the first blocks' one-time work (scratch and ring allocations, twiddle and chirp
  // tables, pinned buffers): run silent blocks through every chain before the source starts. (Not with
  // baseband_write_all, whose sink would record them.)
  if (cfg.input_file_path.empty() && !cfg.baseband_write_all) {
    const size_t block_bytes = cfg.baseband_input_count * static_cast<size_t>(std::abs(cfg.baseband_input_bits)) /
                               srtb::BITS_PER_BYTE * streams;
    auto h_zero = srtb::host_allocator.allocate_shared<std::byte>(block_bytes);
    std::memset(h_zero.get(), 0, block_bytes);
    uint64_t pushed = 0;
    for (int round = 0; round < chains_per_gpu * (blocks_in_flight + 1); round++)
      for (auto& gq : gpu_queues) {
        srtb::work::copy_to_device_work w;
        w.ptr = nullptr;
        w.count = block_bytes;
        w.baseband_data = {h_zero, block_bytes};
        w.timestamp = 0;
        w.udp_packet_counter = w.no_udp_packet_counter;
        w.data_stream_id = 0;
        while (!gq->push(w)) std::this_thread::sleep_for(std::chrono::microseconds(50));
        pushed++;
      }
    while (done->load() < pushed * streams && !g_interrupted) std::this_thread::sleep_for(std::chrono::milliseconds(1));
    done->store(0);
    positives->store(0);
    SRTB_LOGI << " [main] " << "warmed up with " << pushed << " silent block(s)";
  }
  thumbnails_open->store(true);
  const auto t0 = std::chrono::steady_clock::now();
  if (!synth_rate_opt.empty()) {
    // synthetic live stream (BASELINE config #5): one paced receiver, blocks dealt over the GPUs; ends after
    // synthetic_duration seconds of stream and prints one JSON line
    const double rate = std::atof(synth_rate_opt.c_str());
    const std::string fmt{resolve_format_alias(cfg.baseband_format_type)};
    synthetic_stats st;
    std::jthread source;
    if (fmt == "naocpsr_snap1") source = start_synthetic_source<srtb::io::backend_registry::naocpsr_snap1>(0, rate, synth_seconds, rr, st);
    else source = start_synthetic_source<srtb::io::backend_registry::fastmb_roach2>(0, rate, synth_seconds, rr, st);
    source.join();
    while (done->load() < submitted->load() * streams && !g_interrupted) std::this_thread::yield();
    // steady state: from the moment the first assembled block is handed to a GPU (start-up allocations are over) to
    // the last result; the blocks after the first are what arrived in that interval
    const int64_t now_ns = std::chrono::duration_cast<std::chrono::nanoseconds>(
                               std::chrono::steady_clock::now().time_since_epoch()).count();
    const double dt_ = (double)(now_ns - rr.first_ns->load()) * 1e-9;
    const double blocks_in_dt = submitted->load() > 1 ? (double)(submitted->load() - 1) : 0.0;
    std::printf("{\"blocks\": %llu, \"streams\": %zu, \"samples_per_stream_block\": %zu, \"seconds\": %.6f, "
                "\"gsamples_per_s\": %.4f, \"target_samples_per_s\": %.3e, \"received_packets\": %llu, "
                "\"lost_packets\": %llu, \"blocks_with_candidates\": %llu, \"gpus\": %zu}\n",
                (unsigned long long)submitted->load(), streams, (size_t)cfg.baseband_input_count, dt_,
                blocks_in_dt * (double)streams * (double)cfg.baseband_input_count / dt_ / 1e9, rate,
                (unsigned long long)st.received->load(), (unsigned long long)st.lost->load(),
                (unsigned long long)positives->load(), devices.size());
    std::fflush(stdout);
  } else if (!cfg.input_file_path.empty()) {
    std::jthread source = start_pipe<read_file_pipe>(dummy_in_functor<>{}, rr);
    source.join();  // the pipe thread ends when the file has been read
    while (done->load() < submitted->load() * streams && !g_interrupted) std::this_thread::yield();
    // every block has reached the sink, so the side branch has taken all it will: let its thumbnails be written
    while (thumbnails_written->load() < thumbnails_accepted->load() && !g_interrupted)
      std::this_thread::sleep_for(std::chrono::milliseconds(1));
  } else {
    std::vector<std::jthread> sources;
    for (size_t i = 0; i < cfg.udp_receiver_address.size(); i++) {
      const unsigned short port = cfg.udp_receiver_port[std::min(i, cfg.udp_receiver_port.size() - 1)];
      const std::string fmt{resolve_format_alias(cfg.baseband_format_type)};
      if (fmt == "naocpsr_snap1")
        sources.push_back(start_udp_source<srtb::io::backend_registry::naocpsr_snap1>(i, cfg.udp_receiver_address[i], port, rr));
      else if (fmt == "gznupsr_a1")
        sources.push_back(start_udp_source<srtb::io::backend_registry::gznupsr_a1>(i, cfg.udp_receiver_address[i], port, rr));
      else
        sources.push_back(start_udp_source<srtb::io::backend_registry::fastmb_roach2>(i, cfg.udp_receiver_address[i], port, rr));
    }
    while (!g_interrupted) std::this_thread::sleep_for(std::chrono::milliseconds(100));
    for (auto& s : sources) s.request_stop();
  }
  const double dt = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  std::fprintf(stderr, "[srtb_b200] %llu block(s) x %zu stream(s) of %zu samples in %.3f s = %.2f Gsamples/s\n",
               (unsigned long long)submitted->load(), streams, (size_t)cfg.baseband_input_count, dt,
               (double)submitted->load() * (double)streams * (double)cfg.baseband_input_count / dt / 1e9);
  if (cfg.gui_enable)
    std::fprintf(stderr, "[srtb_b200] waterfall: %llu thumbnail(s) written, %llu block(s) skipped while the thumbnail "
                 "pipe was busy\n", (unsigned long long)thumbnails_written->load(),
                 (unsigned long long)thumbnails_dropped->load());
  for (auto& t : threads) t.request_stop();
  threads.clear();
  if (folds) {
    folds->finish();
    SRTB_LOGI << " [main] " << "folded " << folds->blocks() << " block(s) into " << folds->subintegrations()
              << " subintegration(s): " << cfg.baseband_output_file_prefix << "fold.npy"
              << (cfg.fold_coherence ? ", " + cfg.baseband_output_file_prefix + "fold.coherence.npy" : std::string{});
  }
  srtb::device_allocator.deallocate_all_free_ptrs();
  srtb::host_allocator.deallocate_all_free_ptrs();
  return 0;
}
