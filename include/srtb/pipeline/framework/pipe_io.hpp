// srtb/pipeline/framework/pipe_io.hpp — in/out functors connecting pipes to work queues
// (reference: userspace/include/srtb/pipeline/framework/pipe_io.hpp:28-152): blocking queue in/out
// that poll every config.thread_query_work_wait_time ns, a try-once "loose" out, a tee, a container
// splitter and dummies.
#pragma once
#include <chrono>
#include <memory>
#include <optional>
#include <stop_token>
#include <thread>
#include <tuple>

#include "srtb/config.hpp"
#include "srtb/work.hpp"

namespace srtb {
namespace pipeline {

/** how a pipe thread waits on an empty (or full) queue: spin briefly — a block spends tens of microseconds per
 *  stage on the GPU, while sleep_for(1 us) really sleeps ~60 us (timer slack) — then fall back to the reference's
 *  sleep of thread_query_work_wait_time ns (pipe_io.hpp:45). */
struct queue_backoff {
  static constexpr int spin_limit = 2048;
  int spins = 0;
  /** returns true when this wait ended in a real sleep (used to count idle polls) */
  bool wait() {
    if (spins < spin_limit) {
      spins++;
#if defined(__x86_64__) || defined(__i386__)
      __builtin_ia32_pause();
#else
      std::this_thread::yield();
#endif
      return false;
    }
    std::this_thread::sleep_for(std::chrono::nanoseconds(srtb::config.thread_query_work_wait_time));
    return true;
  }
};

template <typename QueuePtr>
class queue_in_functor {
  QueuePtr q_;
  using Work = typename std::pointer_traits<QueuePtr>::element_type::work_type;

 public:
  explicit queue_in_functor(QueuePtr q) : q_{q} {}
  std::optional<Work> operator()(std::stop_token st) {
    Work w;
    queue_backoff backoff;
    while (!q_->pop(w)) {
      if (st.stop_requested()) return std::nullopt;
      backoff.wait();
    }
    return w;
  }
};

/** like queue_in_functor, but hands the pipe a default-constructed work (count == 0: an "idle tick") when nothing
 *  arrived for `idle_polls` polls — lets a pipe that keeps blocks in flight (baseband_chain_pipe) flush them when the
 *  stream pauses or ends. Not in the reference (its pipes hold no state across works). */
template <typename QueuePtr>
class idle_queue_in_functor {
  QueuePtr q_;
  size_t idle_polls_;
  using Work = typename std::pointer_traits<QueuePtr>::element_type::work_type;

 public:
  explicit idle_queue_in_functor(QueuePtr q, size_t idle_polls = 4) : q_{q}, idle_polls_{idle_polls} {}
  std::optional<Work> operator()(std::stop_token st) {
    Work w;
    size_t polls = 0;
    queue_backoff backoff;
    while (!q_->pop(w)) {
      if (st.stop_requested()) return std::nullopt;
      if (polls >= idle_polls_) return Work{};
      if (backoff.wait()) polls++;
    }
    return w;
  }
};

template <typename QueuePtr>
class queue_out_functor {
  QueuePtr q_;
  using Work = typename std::pointer_traits<QueuePtr>::element_type::work_type;

 public:
  explicit queue_out_functor(QueuePtr q) : q_{q} {}
  void operator()(std::stop_token st, Work w) {
    queue_backoff backoff;
    while (!q_->push(w)) {
      if (st.stop_requested()) return;
      backoff.wait();
    }
  }
};

/** push once, drop the work if the queue is full (used for the display side branch) */
template <typename QueuePtr>
class loose_queue_out_functor {
  QueuePtr q_;
  using Work = typename std::pointer_traits<QueuePtr>::element_type::work_type;

 public:
  explicit loose_queue_out_functor(QueuePtr q) : q_{q} {}
  void operator()(std::stop_token st, Work w) {
    if (!st.stop_requested()) q_->push(w);
  }
};

/** copy one work to several out functors */
template <typename... OutFunctors>
class multiple_out_functors_functor {
 public:
  std::tuple<OutFunctors...> out_functors;
  explicit multiple_out_functors_functor(OutFunctors... f) : out_functors{f...} {}
  template <typename Work>
  void operator()(std::stop_token st, Work w) {
    std::apply([&](auto&... f) { (f(st, w), ...); }, out_functors);
  }
};

/** a pipe that returns a container of works (1 in, S out): forward each element */
template <typename OutFunctor>
class multiple_works_out_functor {
 public:
  OutFunctor out_functor;
  explicit multiple_works_out_functor(OutFunctor f) : out_functor{f} {}
  template <typename WorkContainer>
  void operator()(std::stop_token st, WorkContainer works) {
    for (auto&& w : works) {
      if (st.stop_requested()) return;
      out_functor(st, w);
    }
  }
};

template <typename T = srtb::work::dummy_work>
class dummy_in_functor {
 public:
  std::optional<T> operator()(std::stop_token) { return T{}; }
};

template <typename T = srtb::work::dummy_work>
class dummy_out_functor {
 public:
  void operator()(std::stop_token, T) {}
};

}  // namespace pipeline
}  // namespace srtb
