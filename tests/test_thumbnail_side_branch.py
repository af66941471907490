"""Host side of the executable's waterfall branch, no GPU: the side branch's bounded queue drops blocks while the
thumbnail pipe is busy (so it never holds more than its capacity of device spectra), it stays closed until opened, and
the PPM writer replaces the image atomically and leaves the previous image in place when a write fails. A small C++
program over the project's headers is compiled and run."""
import os
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
CUDA = Path(os.environ.get("CUDA_HOME", "/usr/local/cuda"))

PROGRAM = r"""
#include <cassert>
#include <chrono>
#include <cstdio>
#include <fstream>
#include <iterator>
#include <thread>

#include "srtb/pipeline/spectrum_pipe.hpp"

using namespace srtb;

static std::string slurp(const std::string& p) {
  std::ifstream f{p, std::ios::binary};
  return {std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>()};
}

int main(int argc, char** argv) {
  const std::string dir = argv[1];
  // 1. the side branch: closed, then a busy consumer, then room again
  auto q = std::make_shared<pipeline::thumbnail_out_functor::queue>(2);
  auto open = std::make_shared<std::atomic<bool>>(false);
  pipeline::thumbnail_out_functor out{q, open};
  std::stop_source ss;
  work::write_signal_work w;
  w.count = 16;
  w.batch_size = 4;
  w.ptr = std::make_shared<complex<real>>();
  w.baseband_data.baseband_ptr = std::make_shared<std::byte>();
  for (int i = 0; i < 3; i++) out(ss.get_token(), w);
  assert(q->read_available() == 0 && *out.accepted == 0 && *out.dropped == 0);  // warm-up: nothing enters
  open->store(true);
  // a consumer that takes one block and then stays busy for the whole burst
  std::atomic<bool> took{false};
  std::jthread consumer{[&] {
    work::simplify_spectrum_work t;
    while (!q->pop(t)) std::this_thread::yield();
    took = true;
    std::this_thread::sleep_for(std::chrono::milliseconds(200));
  }};
  out(ss.get_token(), w);
  while (!took) std::this_thread::yield();
  for (int i = 0; i < 10; i++) out(ss.get_token(), w);  // the pipe is busy: two queue, eight are dropped
  consumer.join();
  assert(*out.accepted == 3 && *out.dropped == 8 && q->read_available() == 2);
  work::simplify_spectrum_work t;
  assert(q->pop(t) && t.ptr == w.ptr && t.count == 16 && t.batch_size == 4 && !t.baseband_data.baseband_ptr);
  assert(w.ptr.use_count() == 3);  // w, t and the one still queued: nothing else holds the spectrum
  out(ss.get_token(), w);
  assert(*out.accepted == 4 && q->read_available() == 2);

  // 2. the PPM: header, RGB order with alpha dropped, atomic replacement, a failed write keeps the old image
  config.baseband_output_file_prefix = dir + "/run_";
  auto img = std::shared_ptr<uint32_t>(new uint32_t[6]{0xff010203u, 0xff040506u, 0xff070809u,
                                                        0xff0a0b0cu, 0xff0d0e0fu, 0xff101112u},
                                       std::default_delete<uint32_t[]>());
  assert(pipeline::write_waterfall_ppm({img, 7, 3, 2}));
  const std::string path = dir + "/run_waterfall.7.ppm";
  const std::string first = slurp(path);
  assert(first == std::string("P6\n3 2\n255\n") + std::string("\x01\x02\x03\x04\x05\x06\x07\x08\x09\x0a\x0b\x0c"
                                                               "\x0d\x0e\x0f\x10\x11\x12", 18));
  img.get()[0] = 0xff202122u;
  assert(pipeline::write_waterfall_ppm({img, 7, 3, 2}));
  assert(slurp(path).substr(11, 3) == "\x20\x21\x22");
  // the temporary name is taken by a directory: the write fails, the previous image stays
  std::filesystem::create_directory(path + ".tmp");
  img.get()[0] = 0xff303132u;
  assert(!pipeline::write_waterfall_ppm({img, 7, 3, 2}));
  assert(slurp(path).substr(11, 3) == "\x20\x21\x22");
  std::puts("ok");
  return 0;
}
"""


def test_side_branch_drops_while_busy_and_ppm_is_replaced_atomically(tmp_path):
    cxx = shutil.which("g++")
    if cxx is None or not (CUDA / "include" / "cuda_runtime_api.h").exists():
        pytest.skip("needs g++ and the CUDA headers (the executable's build requirements)")
    src = tmp_path / "side_branch.cpp"
    src.write_text(PROGRAM)
    exe = tmp_path / "side_branch"
    subprocess.run([cxx, "-std=c++20", "-O1", "-pthread", "-UNDEBUG", "-I", str(ROOT / "include"), "-I",
                    str(CUDA / "include"), "-o", str(exe), str(src), "-L", str(CUDA / "lib64"), "-lcudart",
                    f"-Wl,-rpath,{CUDA / 'lib64'}"], check=True, capture_output=True, text=True)
    out_dir = tmp_path / "out"
    out_dir.mkdir()
    r = subprocess.run([str(exe), str(out_dir)], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout.strip() == "ok", (r.returncode, r.stdout, r.stderr)
    assert sorted(p.name for p in out_dir.iterdir()) == ["run_waterfall.7.ppm"]  # the failed temporary is removed
