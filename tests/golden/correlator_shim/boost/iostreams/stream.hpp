// boost/iostreams/stream.hpp — host stand-in for the third-party Boost header (see device/file_descriptor.hpp):
// stream<file_descriptor_sink>{path, mode} is an std::ofstream on file_descriptor_sink_path(), whatever `path` says.
#pragma once
#include <fstream>
#include <stdexcept>
#include <string>

#include <boost/iostreams/device/file_descriptor.hpp>

namespace boost {
namespace iostreams {

template <class Device>
class stream : public std::ofstream {
  static const std::string& redirected() {
    const std::string& p = file_descriptor_sink_path();
    if (p.empty()) throw std::runtime_error("boost::iostreams stand-in: no output path set");
    return p;
  }

 public:
  stream(const std::string&, std::ios_base::openmode mode) : std::ofstream(redirected(), mode) {
    if (!is_open()) throw std::runtime_error("boost::iostreams stand-in: cannot open " + redirected());
  }
};

}  // namespace iostreams
}  // namespace boost
