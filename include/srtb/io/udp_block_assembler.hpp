// srtb/io/udp_block_assembler.hpp — packet formats and the counter-keyed block assembler
// (reference: io/backend_registry.hpp:54-153 packet layouts; io/udp/udp_receiver.hpp:180-272
// udp_receive_block_worker): a block holds `expected_packet_count` payloads, packet with counter c
// lands at (c - begin_counter) * payload bytes, packets older than the block are dropped, missing
// packets stay zero (the buffer is zero-filled first), the block closes when a packet with counter
// >= begin + count - 1 arrives and the next block begins at begin + count.
// Differences from the reference: the buffer is zeroed here (the reference relies on its allocator);
// a packet that already belongs to the NEXT block is kept and placed there instead of being dropped
// (the reference discards the packet that closes a block early, :244-251).
// Packet providers: any type with `std::span<const std::byte> receive()`; an in-memory one (synthetic
// "UDP-shaped" streams, BASELINE config #5) and a plain recvfrom() socket one are provided.
#pragma once
#include <chrono>
#include <climits>
#include <cstddef>
#include <cstdint>
#include <cerrno>
#include <cstring>
#include <optional>
#include <span>
#include <stdexcept>
#include <stop_token>
#include <string>
#include <string_view>
#include <vector>

#if __has_include(<sys/socket.h>)
#include <arpa/inet.h>
#include <netinet/in.h>
#include <sys/socket.h>
#include <sys/time.h>
#include <unistd.h>
#define SRTB_HAS_SOCKETS 1
#endif

namespace srtb {
namespace io {
namespace backend_registry {

/** 8-byte little-endian counter + 4096 payload bytes, one stream (backend_registry.hpp:54-73) */
struct fastmb_roach2 {
  static constexpr std::string_view name = "fastmb_roach2";
  static constexpr size_t data_stream_count = 1;
  static constexpr size_t packet_header_size = 8;
  static constexpr size_t packet_payload_size = 4104;  // header + data, as the reference counts it
  static uint64_t parse_counter(std::span<const std::byte> p) {
    uint64_t c = 0;
    for (size_t i = 0; i < 8; i++) c |= static_cast<uint64_t>(p[i]) << (CHAR_BIT * i);
    return c;
  }
  static void write_header(std::span<std::byte> p, uint64_t counter) {
    for (size_t i = 0; i < 8; i++) p[i] = static_cast<std::byte>((counter >> (CHAR_BIT * i)) & 0xff);
  }
};
/** same framing, two polarisations "1 1 2 2" in the payload (backend_registry.hpp:79-85) */
struct naocpsr_snap1 : fastmb_roach2 {
  static constexpr std::string_view name = "naocpsr_snap1";
  static constexpr size_t data_stream_count = 2;
};
/** 32-byte VDIF header + 32 more header bytes, counter = words 6|7 (LE), 8192 payload bytes
 *  (backend_registry.hpp:91-153) */
struct gznupsr_a1 {
  static constexpr std::string_view name = "gznupsr_a1";
  static constexpr size_t data_stream_count = 2;
  static constexpr size_t packet_header_size = 64;
  static constexpr size_t packet_payload_size = 8256;
  static uint64_t parse_counter(std::span<const std::byte> p) {
    uint64_t c = 0;
    for (size_t i = 0; i < 8; i++) c |= static_cast<uint64_t>(p[24 + i]) << (CHAR_BIT * i);  // words 6 and 7
    return c;
  }
  static void write_header(std::span<std::byte> p, uint64_t counter) {
    std::memset(p.data(), 0, packet_header_size);
    for (size_t i = 0; i < 8; i++) p[24 + i] = static_cast<std::byte>((counter >> (CHAR_BIT * i)) & 0xff);
  }
};

}  // namespace backend_registry

namespace udp {

template <typename PacketProvider, typename Backend>
class block_assembler {
 public:
  static constexpr size_t packet_data_size = Backend::packet_payload_size - Backend::packet_header_size;
  PacketProvider provider;
  std::optional<uint64_t> begin_counter;
  size_t total_received_packet_count = 0, total_lost_packet_count = 0;

  explicit block_assembler(PacketProvider p, std::optional<uint64_t> begin = {})
      : provider{std::move(p)}, begin_counter{begin} {}

  /** fill one block; returns the counter of its first packet, or nullopt when the provider is exhausted
   *  before any packet of this block arrived */
  std::optional<uint64_t> receive(std::span<std::byte> block, std::stop_token st = {}) {
    const size_t count = block.size() / packet_data_size;
    if (count * packet_data_size != block.size())
      throw std::invalid_argument{"Packet of size " + std::to_string(packet_data_size) +
                                  " cannot fit into input buffer of size " + std::to_string(block.size())};
    std::memset(block.data(), 0, block.size());
    size_t received = 0;
    bool closed = false;
    auto place = [&](std::span<const std::byte> pkt, uint64_t c) {
      std::memcpy(block.data() + packet_data_size * (c - begin_counter.value()),
                  pkt.data() + Backend::packet_header_size, packet_data_size);
      received++;
    };
    if (carry_.has_value()) {  // a packet past the previous block that arrived while that one was closing
      const uint64_t c = Backend::parse_counter(*carry_);
      if (!begin_counter.has_value()) begin_counter = c;
      if (c >= begin_counter.value() && c < begin_counter.value() + count) place(*carry_, c);
      // a packet more than one block ahead (after a long gap) waits for its own block; this one is all gap
      if (c >= begin_counter.value() + count) closed = true;
      else carry_.reset();
    }
    while (!closed) {
      std::span<const std::byte> pkt;
      if constexpr (requires { provider.receive(st); }) pkt = provider.receive(st);  // live socket: stoppable wait
      else pkt = provider.receive();
      if (pkt.empty()) break;  // provider exhausted (synthetic streams / closed socket / stop requested)
      if (pkt.size() - Backend::packet_header_size != packet_data_size) continue;  // unexpected size: skip
      const uint64_t c = Backend::parse_counter(pkt);
      if (!begin_counter.has_value()) begin_counter = c;
      if (c < begin_counter.value()) continue;  // late packet of an earlier block
      if (c < begin_counter.value() + count) place(pkt, c);
      else carry_storage_.assign(pkt.begin(), pkt.end()), carry_ = std::span<const std::byte>(carry_storage_);
      if (c >= begin_counter.value() + count - 1) closed = true;
    }
    if (received == 0 && !closed) return std::nullopt;
    total_received_packet_count += received;
    total_lost_packet_count += count - received;
    const uint64_t first = begin_counter.value();
    begin_counter = first + count;
    return first;
  }

 private:
  std::vector<std::byte> carry_storage_;
  std::optional<std::span<const std::byte>> carry_;
};

/** packets handed out from a memory buffer, optionally dropping / reordering (tests, synthetic streams) */
class memory_packet_provider {
  std::vector<std::vector<std::byte>> packets_;
  size_t next_ = 0;

 public:
  memory_packet_provider() = default;
  void push(std::vector<std::byte> p) { packets_.push_back(std::move(p)); }
  std::span<const std::byte> receive() {
    if (next_ >= packets_.size()) return {};
    return packets_[next_++];
  }
  size_t remaining() const { return packets_.size() - next_; }
};

/** frame a byte stream into Backend packets with consecutive counters starting at `first_counter` */
template <typename Backend>
inline std::vector<std::vector<std::byte>> frame_stream(std::span<const std::byte> data, uint64_t first_counter) {
  constexpr size_t d = Backend::packet_payload_size - Backend::packet_header_size;
  std::vector<std::vector<std::byte>> out;
  for (size_t off = 0, c = 0; off + d <= data.size(); off += d, c++) {
    std::vector<std::byte> p(Backend::packet_payload_size);
    Backend::write_header(p, first_counter + c);
    std::memcpy(p.data() + Backend::packet_header_size, data.data() + off, d);
    out.push_back(std::move(p));
  }
  return out;
}

/** synthetic LIVE stream (BASELINE config #5): the packets of a few pre-framed blocks are replayed for ever with a
 *  running counter, released at a target payload rate like a NIC would deliver them. A consumer that falls behind by
 *  more than `backlog_bytes` (the socket buffer of a real receiver) loses packets: the counter jumps ahead and the
 *  block assembler zero-fills the gap, exactly as on a real link. rate <= 0: as fast as the consumer takes them. */
template <typename Backend>
class paced_packet_provider {
  static constexpr size_t data_size = Backend::packet_payload_size - Backend::packet_header_size;
  std::vector<std::byte> store_;  // n_ packets of packet_payload_size bytes
  size_t n_ = 0, next_ = 0;
  uint64_t counter_ = 0;
  double bytes_per_s_ = 0;
  size_t backlog_packets_ = 0;
  std::chrono::steady_clock::time_point origin_{};
  bool started_ = false;
  uint64_t released_ = 0;  // packets the "link" has delivered or dropped so far
  uint64_t dropped_ = 0;
  std::chrono::steady_clock::time_point deadline_{};
  double run_seconds_ = 0;  // > 0: stop this long after the first packet was asked for

 public:
  paced_packet_provider(std::span<const std::byte> payload, double payload_bytes_per_s, uint64_t first_counter = 0,
                        size_t backlog_bytes = size_t{64} << 20)
      : counter_{first_counter}, bytes_per_s_{payload_bytes_per_s}, backlog_packets_{backlog_bytes / data_size} {
    n_ = payload.size() / data_size;
    if (n_ == 0) throw std::invalid_argument("[paced_packet_provider] payload smaller than one packet");
    store_.resize(n_ * Backend::packet_payload_size);
    for (size_t i = 0; i < n_; i++)
      std::memcpy(store_.data() + i * Backend::packet_payload_size + Backend::packet_header_size,
                  payload.data() + i * data_size, data_size);
  }
  /** stop handing out packets after `seconds` of stream time (the receiver pipe then ends like a closed socket) */
  void run_for(double seconds) { run_seconds_ = seconds; }
  uint64_t dropped_packets() const { return dropped_; }

  std::span<const std::byte> receive(std::stop_token st = {}) {
    using clock = std::chrono::steady_clock;
    if (!started_) {
      origin_ = clock::now();
      started_ = true;
      deadline_ = origin_ + std::chrono::duration_cast<clock::duration>(std::chrono::duration<double>(run_seconds_));
    }
    const bool has_deadline_ = run_seconds_ > 0;
    if (bytes_per_s_ > 0) {
      for (;;) {
        const auto now = clock::now();
        if (st.stop_requested() || (has_deadline_ && now >= deadline_)) return {};
        const double elapsed = std::chrono::duration<double>(now - origin_).count();
        const uint64_t due = static_cast<uint64_t>(elapsed * bytes_per_s_ / (double)data_size);  // packets sent by now
        if (due > released_ + backlog_packets_) {  // consumer too slow: the oldest packets are gone
          const uint64_t lost = due - released_ - backlog_packets_;
          released_ += lost;
          counter_ += lost;
          next_ = (next_ + lost) % n_;
          dropped_ += lost;
        }
        if (due > released_) break;  // a packet is waiting
        // idle link: nothing has arrived yet
      }
    } else if (st.stop_requested() || (has_deadline_ && clock::now() >= deadline_)) {
      return {};
    }
    std::byte* pkt = store_.data() + next_ * Backend::packet_payload_size;
    Backend::write_header(std::span<std::byte>(pkt, Backend::packet_header_size), counter_);
    next_ = (next_ + 1) % n_;
    counter_++;
    released_++;
    return std::span<const std::byte>(pkt, Backend::packet_payload_size);
  }
};

#ifdef SRTB_HAS_SOCKETS
/** blocking recvfrom() provider (reference: io/udp/recvfrom_packet_provider.hpp) */
class recvfrom_packet_provider {
  int fd_ = -1;
  std::vector<std::byte> buf_;

 public:
  recvfrom_packet_provider(const std::string& address, unsigned short port, size_t max_packet = 9000)
      : buf_(max_packet) {
    fd_ = ::socket(AF_INET, SOCK_DGRAM, 0);
    if (fd_ < 0) throw std::runtime_error("[udp] cannot create socket");
    sockaddr_in addr{};
    addr.sin_family = AF_INET;
    addr.sin_port = htons(port);
    if (::inet_pton(AF_INET, address.c_str(), &addr.sin_addr) != 1) throw std::runtime_error("[udp] bad address " + address);
    int rcvbuf = 64 << 20;
    ::setsockopt(fd_, SOL_SOCKET, SO_RCVBUF, &rcvbuf, sizeof(rcvbuf));
    // bounded blocking: an idle socket must not keep the receiver thread from seeing its stop request
    timeval tv{};
    tv.tv_usec = 100 * 1000;
    ::setsockopt(fd_, SOL_SOCKET, SO_RCVTIMEO, &tv, sizeof(tv));
    if (::bind(fd_, reinterpret_cast<sockaddr*>(&addr), sizeof(addr)) != 0) {
      ::close(fd_);
      fd_ = -1;
      throw std::runtime_error("[udp] bind failed on " + address + ":" + std::to_string(port));
    }
  }
  recvfrom_packet_provider(const recvfrom_packet_provider&) = delete;
  recvfrom_packet_provider& operator=(const recvfrom_packet_provider&) = delete;
  recvfrom_packet_provider(recvfrom_packet_provider&& o) noexcept : fd_{o.fd_}, buf_{std::move(o.buf_)} { o.fd_ = -1; }
  ~recvfrom_packet_provider() {
    if (fd_ >= 0) ::close(fd_);
  }
  /** next datagram; an empty span means "stop requested" (or a socket error), never a mere timeout */
  std::span<const std::byte> receive(std::stop_token st = {}) {
    for (;;) {
      const ssize_t n = ::recvfrom(fd_, buf_.data(), buf_.size(), 0, nullptr, nullptr);
      if (n > 0) return std::span<const std::byte>(buf_.data(), static_cast<size_t>(n));
      if (n < 0 && (errno == EAGAIN || errno == EWOULDBLOCK || errno == EINTR)) {
        if (st.stop_requested()) return {};
        continue;  // idle link: keep listening
      }
      return {};
    }
  }
  /** local port actually bound (port 0 = let the kernel choose; used by the loop-back test) */
  unsigned short bound_port() const {
    sockaddr_in a{};
    socklen_t len = sizeof(a);
    if (::getsockname(fd_, reinterpret_cast<sockaddr*>(&a), &len) != 0) return 0;
    return ntohs(a.sin_port);
  }
};
#endif

}  // namespace udp
}  // namespace io
}  // namespace srtb
