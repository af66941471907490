// srtb/program_options.hpp — config loader with the reference's semantics
// (reference: userspace/include/srtb/program_options.hpp:34-309): every numeric option is an
// arithmetic EXPRESSION string ("2 ** 30", "1405 + (64 / 2)", "128 * 1e6") evaluated to double and
// cast to the field type (:197-214); list options are split on ',' (:223-250); priority is
// command line > config file > defaults (:148-173). Boost.Program_options / Boost.Spirit are not
// used: a small recursive-descent evaluator implements the grammar of the vendored exprgrammar
// (3rdparty/exprgrammar/include/suzerain/exprgrammar.hpp:203-231):
//   expression = term (('+'|'-') term)* ; term = factor (('*'|'/') factor)* ;
//   factor = primary ('**' factor)* ; primary = real | '(' expression ')' | '-' primary | '+' primary
//          | ufunc '(' expression ')' | bfunc '(' expression ',' expression ')' | constant
// (names case-insensitive; constants digits, digits10, e, epsilon, pi).
#pragma once
#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstdlib>
#include <filesystem>
#include <fstream>
#include <limits>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>

#include "srtb/config.hpp"
#include "srtb/log.hpp"

namespace srtb {
namespace program_options {

class expression_parser {
  const char* p_;
  const char* end_;

  void skip() {
    while (p_ < end_ && std::isspace(static_cast<unsigned char>(*p_))) p_++;
  }
  bool eat(char c) {
    skip();
    if (p_ < end_ && *p_ == c) {
      p_++;
      return true;
    }
    return false;
  }
  [[noreturn]] void fail(const std::string& why) const {
    throw std::invalid_argument("[program_options] cannot parse expression: " + why);
  }
  std::string ident() {
    skip();
    std::string s;
    while (p_ < end_ && (std::isalnum(static_cast<unsigned char>(*p_)) || *p_ == '_'))
      s.push_back(static_cast<char>(std::tolower(static_cast<unsigned char>(*p_++))));
    return s;
  }
  double primary() {
    skip();
    if (p_ >= end_) fail("unexpected end");
    if (eat('(')) {
      const double v = expression();
      if (!eat(')')) fail("missing ')'");
      return v;
    }
    if (eat('-')) return -primary();
    if (eat('+')) return primary();
    if (std::isdigit(static_cast<unsigned char>(*p_)) || *p_ == '.') {
      char* after = nullptr;
      const double v = std::strtod(p_, &after);
      if (after == p_) fail("bad number");
      p_ = after;
      return v;
    }
    const std::string name = ident();
    if (name.empty()) fail(std::string("unexpected character '") + *p_ + "'");
    static const std::map<std::string, double (*)(double)> ufunc = {
        {"abs", [](double x) { return std::abs(x); }},   {"acos", [](double x) { return std::acos(x); }},
        {"asin", [](double x) { return std::asin(x); }}, {"atan", [](double x) { return std::atan(x); }},
        {"ceil", [](double x) { return std::ceil(x); }}, {"cos", [](double x) { return std::cos(x); }},
        {"cosh", [](double x) { return std::cosh(x); }}, {"exp", [](double x) { return std::exp(x); }},
        {"floor", [](double x) { return std::floor(x); }}, {"log", [](double x) { return std::log(x); }},
        {"log10", [](double x) { return std::log10(x); }}, {"sin", [](double x) { return std::sin(x); }},
        {"sinh", [](double x) { return std::sinh(x); }}, {"sqrt", [](double x) { return std::sqrt(x); }},
        {"tan", [](double x) { return std::tan(x); }},   {"tanh", [](double x) { return std::tanh(x); }}};
    static const std::map<std::string, double (*)(double, double)> bfunc = {
        {"atan2", [](double a, double b) { return std::atan2(a, b); }},
        {"max", [](double a, double b) { return std::max(a, b); }},
        {"min", [](double a, double b) { return std::min(a, b); }},
        {"pow", [](double a, double b) { return std::pow(a, b); }}};
    if (auto it = ufunc.find(name); it != ufunc.end()) {
      if (!eat('(')) fail("missing '(' after " + name);
      const double a = expression();
      if (!eat(')')) fail("missing ')'");
      return it->second(a);
    }
    if (auto it = bfunc.find(name); it != bfunc.end()) {
      if (!eat('(')) fail("missing '(' after " + name);
      const double a = expression();
      if (!eat(',')) fail("missing ','");
      const double b = expression();
      if (!eat(')')) fail("missing ')'");
      return it->second(a, b);
    }
    if (name == "pi") return 3.141592653589793238462643383279502884;
    if (name == "e") return 2.718281828459045235360287471352662498;
    if (name == "epsilon") return std::numeric_limits<double>::epsilon();
    if (name == "digits") return std::numeric_limits<double>::digits;
    if (name == "digits10") return std::numeric_limits<double>::digits10;
    fail("unknown name '" + name + "'");
  }
  double factor() {
    double v = primary();
    skip();
    while (p_ + 1 < end_ && p_[0] == '*' && p_[1] == '*') {
      p_ += 2;
      v = std::pow(v, factor());
      skip();
    }
    return v;
  }
  double term() {
    double v = factor();
    while (true) {
      skip();
      if (p_ < end_ && *p_ == '*' && !(p_ + 1 < end_ && p_[1] == '*')) {
        p_++;
        v *= factor();
      } else if (p_ < end_ && *p_ == '/') {
        p_++;
        v /= factor();
      } else {
        return v;
      }
    }
  }
  double expression() {
    double v = term();
    while (true) {
      if (eat('+')) v += term();
      else if (eat('-')) v -= term();
      else return v;
    }
  }

 public:
  explicit expression_parser(const std::string& s) : p_{s.data()}, end_{s.data() + s.size()} {}
  double parse_all() {
    const double v = expression();
    skip();
    if (p_ != end_) fail(std::string("trailing characters \"") + p_ + "\"");
    return v;
  }
};

/** evaluate a constant arithmetic expression (program_options.hpp:188-192) */
inline double parse(const std::string& expression) { return expression_parser{expression}.parse_all(); }

inline std::string trim(const std::string& s) {
  size_t a = 0, b = s.size();
  while (a < b && std::isspace(static_cast<unsigned char>(s[a]))) a++;
  while (b > a && std::isspace(static_cast<unsigned char>(s[b - 1]))) b--;
  return s.substr(a, b - a);
}

/** split on a delimiter with adjacent delimiters compressed (boost::split + token_compress_on) */
inline std::vector<std::string> split_list(const std::string& value, char delimiter) {
  std::vector<std::string> out(1);
  bool prev = false;
  for (char c : value) {
    if (c == delimiter) {
      if (!prev) out.emplace_back();
      prev = true;
    } else {
      out.back().push_back(c);
      prev = false;
    }
  }
  return out;
}

/** the trial DMs of a dm_list value, in the order given: comma-separated items, each one expression ("2 * 281.025")
 *  or a range start:stop:step of expressions, which expands to start + i * step for i = 0 .. floor((stop - start) /
 *  step + 0.5), computed in double from i. An empty list gives no trials; an empty item, a non-finite value, a
 *  step <= 0 or a stop < start throws std::invalid_argument naming the key. */
inline std::vector<srtb::real> parse_dm_list(const std::string& value) {
  std::vector<srtb::real> out;
  if (trim(value).empty()) return out;
  auto bad = [&](const std::string& why) -> std::invalid_argument {
    return std::invalid_argument("[program_options] dm_list = \"" + value + "\": " + why);
  };
  auto eval = [&](const std::string& s) {
    if (trim(s).empty()) throw bad("empty item");
    double v = 0;
    try {
      v = parse(s);
    } catch (const std::invalid_argument& e) {
      throw bad(e.what());
    }
    if (!std::isfinite(v)) throw bad("\"" + trim(s) + "\" is not finite");
    return v;
  };
  size_t pos = 0;
  while (true) {
    const size_t comma = value.find(',', pos);
    const std::string item = value.substr(pos, comma == std::string::npos ? std::string::npos : comma - pos);
    if (item.find(':') == std::string::npos) {
      out.push_back(static_cast<srtb::real>(eval(item)));
    } else {
      std::vector<std::string> parts;
      size_t p = 0;
      while (true) {
        const size_t colon = item.find(':', p);
        parts.push_back(item.substr(p, colon == std::string::npos ? std::string::npos : colon - p));
        if (colon == std::string::npos) break;
        p = colon + 1;
      }
      if (parts.size() != 3) throw bad("range \"" + trim(item) + "\" is not start:stop:step");
      const double start = eval(parts[0]), stop = eval(parts[1]), step = eval(parts[2]);
      if (!(step > 0)) throw bad("range \"" + trim(item) + "\" has step <= 0");
      if (stop < start) throw bad("range \"" + trim(item) + "\" has stop < start");
      const double count = std::floor((stop - start) / step + 0.5);
      for (double i = 0; i <= count; i++) out.push_back(static_cast<srtb::real>(start + i * step));
    }
    if (comma == std::string::npos) break;
    pos = comma + 1;
  }
  return out;
}

/** "key = value" lines, '#' comments; unknown keys are rejected like Boost.Program_options does */
inline const std::vector<std::string>& known_options() {
  static const std::vector<std::string> names = {
      "config_file_name", "log_level", "thread_query_work_wait_time", "gui_enable", "gui_pixmap_width",
      "gui_pixmap_height", "baseband_input_count", "baseband_input_bits", "baseband_format_type",
      "baseband_freq_low", "baseband_bandwidth", "baseband_sample_rate", "baseband_reserve_sample",
      "udp_receiver_address", "udp_receiver_port", "udp_receiver_cpu_preferred", "input_file_path",
      "input_file_offset_bytes", "baseband_output_file_prefix", "baseband_write_all", "dm", "dm_list",
      "incoherent_dm_list",
      "dedisperse_measurement", "fft_fftw_wisdom_path", "mitigate_rfi_average_method_threshold",
      "mitigate_rfi_spectral_kurtosis_threshold", "mitigate_rfi_freq_list", "spectrum_channel_count",
      "signal_detect_signal_noise_threshold", "signal_detect_channel_threshold", "signal_detect_max_boxcar_length",
      "signal_detect_sum_polarizations", "fold_period", "fold_period_derivative", "fold_bin_count",
      "fold_subband_count", "fold_subintegration_blocks", "fold_coherence", "dm_search_candidates",
      "signal_detect_candidates", "candidate_cutouts"};
  return names;
}

inline void check_known(const std::string& key) {
  const auto& n = known_options();
  if (std::find(n.begin(), n.end(), key) == n.end())
    throw std::invalid_argument("[program_options] unrecognised option '" + key + "'");
}

inline std::map<std::string, std::string> parse_config_text(const std::string& text) {
  std::map<std::string, std::string> out;
  size_t pos = 0;
  while (pos <= text.size()) {
    size_t nl = text.find('\n', pos);
    if (nl == std::string::npos) nl = text.size();
    std::string line = text.substr(pos, nl - pos);
    pos = nl + 1;
    if (const size_t hash = line.find('#'); hash != std::string::npos) line.resize(hash);
    line = trim(line);
    if (line.empty()) continue;
    const size_t eq = line.find('=');
    if (eq == std::string::npos) throw std::invalid_argument("[program_options] invalid config line: " + line);
    std::string key = trim(line.substr(0, eq));
    check_known(key);
    if (key == "dedisperse_measurement") key = "dm";
    out[key] = trim(line.substr(eq + 1));
  }
  return out;
}

/** command line (--key value | --key=value) over config file over defaults */
[[nodiscard]] inline std::map<std::string, std::string> parse_arguments(int argc, char** argv,
                                                                         const std::string& default_config_file_name) {
  std::map<std::string, std::string> cmd;
  for (int i = 1; i < argc; i++) {
    std::string a = argv[i];
    if (a.rfind("--", 0) != 0) throw std::invalid_argument("[program_options] unexpected argument '" + a + "'");
    a = a.substr(2);
    std::string key, value;
    if (const size_t eq = a.find('='); eq != std::string::npos) {
      key = a.substr(0, eq);
      value = a.substr(eq + 1);
    } else {
      key = a;
      if (i + 1 >= argc) throw std::invalid_argument("[program_options] option '--" + key + "' needs a value");
      value = argv[++i];
    }
    check_known(key);
    if (key == "dedisperse_measurement") key = "dm";
    cmd[key] = value;
  }
  const std::string file = cmd.count("config_file_name") ? cmd["config_file_name"] : default_config_file_name;
  std::map<std::string, std::string> merged;
  if (std::filesystem::exists(file)) {
    SRTB_LOGI << " [program_options] " << "using config file " << file;
    std::ifstream f(file);
    const std::string text((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    merged = parse_config_text(text);
  } else {
    SRTB_LOGW << " [program_options] " << "config file " << file << " not found.";
  }
  for (auto& kv : cmd) merged[kv.first] = kv.second;  // command line wins
  return merged;
}

inline void evaluate_and_apply_changed_config(const std::string& name, const std::string& value,
                                              srtb::configs& config) {
#define SRTB_PARSE(target_name)                                                                   \
  if (name == #target_name) {                                                                     \
    using target_type = decltype(config.target_name);                                             \
    config.target_name = static_cast<target_type>(parse(value));                                  \
    SRTB_LOGI << " [program_options] " << #target_name << " = " << config.target_name;            \
    return;                                                                                       \
  }
#define SRTB_ASSIGN(target_name)                                                 \
  if (name == #target_name) {                                                    \
    config.target_name = value;                                                  \
    SRTB_LOGI << " [program_options] " << #target_name << " = " << value;        \
    return;                                                                      \
  }
#define SRTB_SPLIT_PARSE(target_name)                                                    \
  if (name == #target_name) {                                                            \
    using target_type = typename decltype(config.target_name)::value_type;              \
    config.target_name.clear();                                                          \
    for (const auto& sub : split_list(value, ','))                                       \
      config.target_name.push_back(static_cast<target_type>(parse(sub)));                \
    return;                                                                              \
  }
  SRTB_PARSE(baseband_input_count)
  SRTB_PARSE(baseband_input_bits)
  SRTB_ASSIGN(baseband_format_type)
  SRTB_PARSE(baseband_freq_low)
  SRTB_PARSE(baseband_bandwidth)
  SRTB_PARSE(baseband_sample_rate)
  SRTB_PARSE(baseband_reserve_sample)
  SRTB_PARSE(dm)
  if (name == "dm_list") {
    const auto trials = parse_dm_list(value);  // rejects a bad list here, before any pipe starts
    config.dm_list = value;
    SRTB_LOGI << " [program_options] " << "dm_list = " << value << " (" << trials.size() << " trial(s))";
    return;
  }
  if (name == "incoherent_dm_list") {
    std::vector<srtb::real> trials;
    try {
      trials = parse_dm_list(value);  // the same syntax; a bad list is rejected here, named by its own key
    } catch (const std::invalid_argument& e) {
      throw std::invalid_argument(std::string{"[program_options] incoherent_dm_list: "} + e.what());
    }
    config.incoherent_dm_list = value;
    SRTB_LOGI << " [program_options] " << "incoherent_dm_list = " << value << " (" << trials.size() << " trial(s))";
    return;
  }
  if (name == "udp_receiver_address") {
    config.udp_receiver_address.clear();
    for (const auto& sub : split_list(value, ',')) config.udp_receiver_address.push_back(trim(sub));
    return;
  }
  SRTB_SPLIT_PARSE(udp_receiver_port)
  SRTB_SPLIT_PARSE(udp_receiver_cpu_preferred)
  SRTB_ASSIGN(input_file_path)
  SRTB_PARSE(input_file_offset_bytes)
  SRTB_ASSIGN(baseband_output_file_prefix)
  SRTB_PARSE(baseband_write_all)
  SRTB_ASSIGN(fft_fftw_wisdom_path)
  SRTB_PARSE(mitigate_rfi_average_method_threshold)
  SRTB_PARSE(mitigate_rfi_spectral_kurtosis_threshold)
  SRTB_ASSIGN(mitigate_rfi_freq_list)
  SRTB_PARSE(spectrum_channel_count)
  SRTB_PARSE(signal_detect_signal_noise_threshold)
  SRTB_PARSE(signal_detect_channel_threshold)
  SRTB_PARSE(signal_detect_max_boxcar_length)
  SRTB_PARSE(signal_detect_sum_polarizations)
  SRTB_PARSE(fold_period)
  SRTB_PARSE(fold_period_derivative)
  SRTB_PARSE(fold_bin_count)
  SRTB_PARSE(fold_subband_count)
  SRTB_PARSE(fold_subintegration_blocks)
  SRTB_PARSE(fold_coherence)
  SRTB_PARSE(dm_search_candidates)
  SRTB_PARSE(signal_detect_candidates)
  SRTB_PARSE(candidate_cutouts)
  SRTB_PARSE(thread_query_work_wait_time)
  SRTB_PARSE(gui_enable)
  SRTB_PARSE(gui_pixmap_width)
  SRTB_PARSE(gui_pixmap_height)
  SRTB_ASSIGN(config_file_name)
  if (name == "log_level") {  // program_options.hpp:282-288
    srtb::log::current_level = static_cast<srtb::log::levels>(static_cast<int>(parse(value)));
    return;
  }
#undef SRTB_PARSE
#undef SRTB_ASSIGN
#undef SRTB_SPLIT_PARSE
  SRTB_LOGW << " [program_options] " << "Unrecognized config: name = " << name << ", value = " << value;
}

/** a coherent DM sweep (dm_list) and an incoherent search around dm (incoherent_dm_list) are two ways to search one
 *  block; both set is rejected, naming both keys */
inline void check_dm_search_keys(const srtb::configs& config) {
  if (!trim(config.dm_list).empty() && !trim(config.incoherent_dm_list).empty())
    throw std::invalid_argument(
        "[program_options] dm_list and incoherent_dm_list are both set: choose the coherent DM sweep (dm_list) or the "
        "incoherent search around dm (incoherent_dm_list)");
}

/** dm_search_candidates lists the candidates of a DM search: it needs one (dm_list or incoherent_dm_list) */
inline void check_dm_search_candidates(const srtb::configs& config) {
  if (config.dm_search_candidates && trim(config.dm_list).empty() && trim(config.incoherent_dm_list).empty())
    throw std::invalid_argument("[program_options] dm_search_candidates needs a DM search: set dm_list (the coherent "
                                "DM sweep) or incoherent_dm_list (the incoherent search around dm)");
}

/** signal_detect_candidates lists the block path's candidates; a DM search (dm_list, incoherent_dm_list) lists its own
 *  through dm_search_candidates, so the two are not combined */
inline void check_signal_detect_candidates(const srtb::configs& config) {
  if (config.signal_detect_candidates && (!trim(config.dm_list).empty() || !trim(config.incoherent_dm_list).empty()))
    throw std::invalid_argument("[program_options] signal_detect_candidates lists the candidates of the block path at "
                                "its one dm; with dm_list or incoherent_dm_list set, use dm_search_candidates instead");
}

/** candidate_cutouts cuts out candidates a candidate list names: it needs one (signal_detect_candidates or
 *  dm_search_candidates), is a count (not negative), and needs the spectrum of each candidate's block, which the
 *  coherent DM sweep (dm_list) keeps for no trial */
inline void check_candidate_cutouts(const srtb::configs& config) {
  if (config.candidate_cutouts < 0)
    throw std::invalid_argument("[program_options] candidate_cutouts is a count of candidates per file: got " +
                                std::to_string(config.candidate_cutouts));
  if (config.candidate_cutouts == 0) return;
  if (!config.signal_detect_candidates && !config.dm_search_candidates)
    throw std::invalid_argument("[program_options] candidate_cutouts needs a candidate list: set "
                                "signal_detect_candidates (the block path) or dm_search_candidates (a DM search)");
  if (!trim(config.dm_list).empty())
    throw std::invalid_argument("[program_options] candidate_cutouts is not available with dm_list: the coherent DM "
                                "sweep keeps no trial's spectrum; use incoherent_dm_list");
}

/** signal_detect_sum_polarizations adds the streams of a block: it needs two or more (`streams`, the format's count),
 *  and it is a block-path detector, so neither DM search (dm_list, incoherent_dm_list) takes it */
inline void check_sum_polarizations(const srtb::configs& config, size_t streams) {
  if (!config.signal_detect_sum_polarizations) return;
  if (streams < 2)
    throw std::invalid_argument("[program_options] signal_detect_sum_polarizations needs a format with two or more "
                                "streams, but baseband_format_type = " + config.baseband_format_type + " has " +
                                std::to_string(streams));
  if (!trim(config.dm_list).empty())
    throw std::invalid_argument("[program_options] signal_detect_sum_polarizations and dm_list are both set: the "
                                "coherent DM sweep has no total-intensity detector");
  if (!trim(config.incoherent_dm_list).empty())
    throw std::invalid_argument("[program_options] signal_detect_sum_polarizations and incoherent_dm_list are both set: "
                                "the incoherent search has no total-intensity detector");
}

/** folding (fold_period != 0) at start-up: a finite, positive period of at least two spectrum samples (2 dt, dt =
 *  2C / baseband_sample_rate with C = min(spectrum_channel_count, baseband_input_count / 2)), 1 to 4096 bins, a subband
 *  count that divides C, no dm_list (the sweep gives each stream another DM) and a recording to fold (input_file_path);
 *  fold_coherence needs fold_period and a two-stream format: naocpsr_snap1, interleaved_samples_2 or gznupsr_a1 */
inline void check_fold(const srtb::configs& config) {
  if (config.fold_coherence) {  // the coherence products pair the two feeds of a dual-polarisation format
    if (config.fold_period == 0)
      throw std::invalid_argument("[program_options] fold_coherence needs fold_period: it folds at the fold's period");
    const std::string& f = config.baseband_format_type;
    if (f == "gznupsr_a1_4")
      throw std::invalid_argument("[program_options] fold_coherence with baseband_format_type = gznupsr_a1_4: its four "
                                  "streams are not documented as two feed pairs");
    if (f != "naocpsr_snap1" && f != "interleaved_samples_2" && f != "gznupsr_a1")
      throw std::invalid_argument("[program_options] fold_coherence with baseband_format_type = " + f +
                                  ": a single-stream format has no second polarisation to pair");
  }
  if (config.fold_period == 0) return;
  const double P = config.fold_period;
  if (!std::isfinite(P) || P < 0 || !std::isfinite(config.fold_period_derivative))
    throw std::invalid_argument("[program_options] fold_period = " + std::to_string(P) + ", fold_period_derivative = " +
                                std::to_string(config.fold_period_derivative) +
                                ": the period must be finite and positive, its derivative finite");
  const size_t C = std::min<size_t>(config.spectrum_channel_count, config.baseband_input_count / 2);
  const double dt = 2.0 * (double)C / (double)config.baseband_sample_rate;
  if (!(P >= 2 * dt))
    throw std::invalid_argument("[program_options] fold_period = " + std::to_string(P) +
                                " s is shorter than two spectrum samples (2 dt = " + std::to_string(2 * dt) +
                                " s; dt = 2 spectrum_channel_count / baseband_sample_rate)");
  if (config.fold_bin_count < 1 || config.fold_bin_count > 4096)
    throw std::invalid_argument("[program_options] fold_bin_count = " + std::to_string(config.fold_bin_count) +
                                " is outside 1..4096");
  if (config.fold_subband_count == 0 || C % config.fold_subband_count)
    throw std::invalid_argument("[program_options] fold_subband_count = " + std::to_string(config.fold_subband_count) +
                                " does not divide the " + std::to_string(C) + " channels (spectrum_channel_count)");
  if (!trim(config.dm_list).empty())
    throw std::invalid_argument("[program_options] fold_period and dm_list are both set: the DM sweep hands out a "
                                "different DM per stream, fold at one dm instead");
  if (trim(config.input_file_path).empty())
    throw std::invalid_argument("[program_options] fold_period needs input_file_path: only recordings are folded");
}

inline void apply_changed_configs(const std::map<std::string, std::string>& changed, srtb::configs& config) {
  for (const auto& [name, value] : changed) evaluate_and_apply_changed_config(name, value, config);
  check_dm_search_keys(config);
}

}  // namespace program_options
}  // namespace srtb
