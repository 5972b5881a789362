// TEST INFRASTRUCTURE ONLY -- the per-ray arithmetic of the irradiance binning kernel (csrc/olb_irradiance.cuh)
// compiled for the host, so that its bin choice can be compared with np.histogram2d without a GPU.  Built as its own
// library (_hostcheck_irradiance.so, oracle/hostcheck_irradiance.py); never linked into libolb.so.
#include "../../include/olb.h"
#include "../../optiland_b200/csrc/olb_irradiance.cuh"

using namespace olb;

template <typename T>
static void run(const T* x, const T* y, const T* z, const T* i, int64_t n, int32_t frame, const double* t,
                const double* R, const double* xe, int32_t nx, const double* ye, int32_t ny, int64_t* bins, double* hist) {
  IrrFrame f;
  f.affine = frame == OLB_IRR_FRAME_AFFINE;
  for (int k = 0; k < 3; ++k) f.t[k] = t[k];
  for (int k = 0; k < 9; ++k) f.R[k] = f.affine ? R[k] : (k % 4 == 0 ? 1.0 : 0.0);
  const double x_inv = nx / (xe[nx] - xe[0]), y_inv = ny / (ye[ny] - ye[0]);
  for (int64_t r = 0; r < n; ++r) {
    const int64_t b = irr_ray_bin<T>(x[r], y[r], f.affine ? z[r] : (T)0, i[r], f, xe, nx, x_inv, ye, ny, y_inv);
    bins[r] = b;
    if (b >= 0) hist[b] += (double)i[r];
  }
}

extern "C" {
// bins[r]: the flat bin ix * ny + iy ray r lands in, or -1; hist (nx * ny) is accumulated into
void olbhc_irradiance_f64(const double* x, const double* y, const double* z, const double* i, int64_t n, int32_t frame,
                          const double* t, const double* R, const double* xe, int32_t nx, const double* ye, int32_t ny,
                          int64_t* bins, double* hist) {
  run<double>(x, y, z, i, n, frame, t, R, xe, nx, ye, ny, bins, hist);
}
void olbhc_irradiance_f32(const float* x, const float* y, const float* z, const float* i, int64_t n, int32_t frame,
                          const double* t, const double* R, const double* xe, int32_t nx, const double* ye, int32_t ny,
                          int64_t* bins, double* hist) {
  run<float>(x, y, z, i, n, frame, t, R, xe, nx, ye, ny, bins, hist);
}
}
