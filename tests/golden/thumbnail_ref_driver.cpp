// thumbnail_ref_driver.cpp — runs the REFERENCE'S OWN waterfall thumbnail operators (resample_spectrum_3,
// simplify_spectrum_normalize_with_average_value, generate_pixmap of srtb/spectrum/simplify_spectrum.hpp) through the
// host SYCL shim of oracle/ref_shim, compiled from the reference tree where it lies (nothing is copied). Used only by
// make_thumbnail_golden.py to write srtb_thumbnail_ref_vectors.npz.
//
// The operators ask the device for three things the shim does not declare; they are added here, before the
// reference's headers are read: info::device::sub_group_sizes (the shim answers {32, 32, 32}, so the smallest
// sub-group is 32), max_work_item_sizes<1> as an id<1>, and the three-argument local_accessor (range, handler, no_init);
// and sycl::ceil / sycl::floor, which call the f-suffixed libm functions as the shim's other math does.
#include <sycl/sycl.hpp>

namespace sycl {
struct no_init_t {};
inline constexpr no_init_t no_init{};
namespace info {
namespace device {
struct sub_group_sizes {
  using return_type = std::vector<size_t>;
};
template <>
struct max_work_item_sizes<1> {
  using return_type = id<1>;
};
}  // namespace device
}  // namespace info
template <>
struct local_accessor<float, 1> {
  std::shared_ptr<std::vector<float>> store;
  local_accessor(range<1> r, handler&) : store{std::make_shared<std::vector<float>>(r.size())} {}
  local_accessor(range<1> r, handler&, no_init_t) : store{std::make_shared<std::vector<float>>(r.size())} {}
  float& operator[](size_t i) const { return (*store)[i]; }
};
inline float ceil(float x) { return ::ceilf(x); }
inline double ceil(double x) { return ::ceil(x); }
inline float floor(float x) { return ::floorf(x); }
inline double floor(double x) { return ::floor(x); }
}  // namespace sycl

#include <cstdint>
#include <cstring>
#include <vector>

#include "srtb/commons.hpp"
#include "srtb/spectrum/simplify_spectrum.hpp"  // reference operator header (verbatim)

extern "C" {

// spec: [in_height][in_width] complex64; raw: resampled intensity before normalisation; inten: after; pixmap: ARGB32
int srtb_ref_simplify_spectrum(const float* spec, size_t in_width, size_t in_height, size_t out_width,
                               size_t out_height, float* raw, float* inten, uint32_t* pixmap, float* average) {
  using C = srtb::complex<srtb::real>;
  static sycl::queue q;
  std::vector<C> in(in_width * in_height);
  std::memcpy(in.data(), spec, sizeof(C) * in.size());
  const size_t n = out_width * out_height;
  std::vector<srtb::real> out(n);
  srtb::spectrum::resample_spectrum_3(
      in.data(), in_width, in_height, [](auto&& x) { return srtb::norm(x); }, out.data(), out_width, out_height, q);
  std::memcpy(raw, out.data(), sizeof(float) * n);
  *average = srtb::spectrum::simplify_spectrum_normalize_with_average_value(out.data(), n, q);
  std::memcpy(inten, out.data(), sizeof(float) * n);
  srtb::spectrum::generate_pixmap(out.data(), pixmap, out_width, out_height, srtb::gui::color_0, srtb::gui::color_1,
                                  srtb::gui::color_overflow, q);
  return 0;
}

}  // extern "C"
