// boost/iostreams/device/file_descriptor.hpp — host stand-in for the third-party Boost header, for the reference's
// correlator.cpp only (tests/golden/correlator_ref_driver.cpp). A file_descriptor_sink does not open the path the
// program names: every sink opens the path the driver sets in file_descriptor_sink_path(), and an unset path refuses
// to open anything, so a golden run never writes to the reference's /dev/shm/corr.bin.
#pragma once
#include <ios>
#include <string>

#define BOOST_IOS std::ios_base

namespace boost {
namespace iostreams {

inline std::string& file_descriptor_sink_path() {
  static std::string path;
  return path;
}

struct file_descriptor_sink {};

}  // namespace iostreams
}  // namespace boost
