// correlator_ref_driver.cpp — runs the REFERENCE'S OWN baseband correlator (userspace/src/correlator.cpp), compiled
// unmodified from the reference tree where it lies (nothing is copied) through the host SYCL shim of oracle/ref_shim
// and the boost::iostreams stand-ins next to this file (correlator_shim/). With no vendor FFT in the shim, the
// reference's FFT dispatcher takes its naive_fft. Used only by make_correlator_golden.py to write
// srtb_correlator_ref_vectors.npz.
//
//   correlator_ref_driver <output file>
//
// reads pol_1.bin and pol_2.bin in the working directory, as the reference does, and writes its raw float32 output to
// <output file> instead of /dev/shm/corr.bin.
#include <boost/iostreams/device/file_descriptor.hpp>
#include <cstdio>

#define main srtb_ref_correlator_main
#include "correlator.cpp"  // the reference's, found through -I <reference>/src
#undef main

int main(int argc, char** argv) {
  if (argc != 2) {
    std::fprintf(stderr, "usage: %s <output file>\n", argv[0]);
    return 2;
  }
  boost::iostreams::file_descriptor_sink_path() = argv[1];
  return srtb_ref_correlator_main();
}
