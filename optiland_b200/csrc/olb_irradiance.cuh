// olb_irradiance.cuh -- per-ray arithmetic of the irradiance binning kernel (olb_irradiance.cu).
//
// Reference: IncoherentIrradiance._generate_field_data, non-differentiable branch (optiland/analysis/irradiance.py:
// 294-353): localize the ray points into the detector's frame (visualization/system/utils.py:16-46 ->
// CoordinateSystem.localize), keep power > 0, np.histogram2d with the power as weights.  Semantics: include/olb.h,
// OlbIrradiance.
//
// Shared by olb_irradiance.cu (device) and tests/hostcheck/hostcheck_irradiance.cpp (g++; TEST INFRASTRUCTURE), so
// that the bin choice can be compared with np.histogram2d in the GPU-less build container.
#ifndef OLB_IRRADIANCE_CUH_
#define OLB_IRRADIANCE_CUH_
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define OLB_IRR_HD __host__ __device__ __forceinline__
#else
#define OLB_IRR_HD inline
#endif

namespace olb {

struct IrrFrame {
  int32_t affine;   // OLB_IRR_FRAME_AFFINE
  double t[3];
  double R[9];      // row-major
};

// searchsorted(e, v, side="right") - 1 over the n + 1 strictly increasing edges e, with v == e[n] in the last bin;
// -1 for v outside [e[0], e[n]] and for NaN.  The guess from the mean pitch is exact for linspace / arange edges up
// to rounding; the two walks make it exact for any increasing edges.
OLB_IRR_HD int32_t irr_bin(double v, const double* e, int32_t n, double inv_pitch) {
  if (!(v >= e[0] && v <= e[n])) return -1;
  if (v == e[n]) return n - 1;
  double g = (v - e[0]) * inv_pitch;
  int32_t k = g < (double)(n - 1) ? (int32_t)g : n - 1;
  while (k > 0 && v < e[k]) --k;
  while (k < n - 1 && v >= e[k + 1]) ++k;
  return k;
}

// r * v, or 0 for a zero entry (a rotation by a zero angle is skipped by the reference, so an infinite coordinate
// along an axis the frame does not mix in stays out of the sum)
OLB_IRR_HD double irr_term(double acc, double r, double v) { return r != 0.0 ? fma(r, v, acc) : acc; }

// Local (x, y) of one ray point.  Translation-only frames subtract in the ray's own precision T.
template <typename T>
OLB_IRR_HD void irr_localize(T x, T y, T z, const IrrFrame& f, double& xl, double& yl) {
  if (!f.affine) {
    xl = (double)(x - (T)f.t[0]);
    yl = (double)(y - (T)f.t[1]);
    return;
  }
  const double dx = (double)x - f.t[0], dy = (double)y - f.t[1], dz = (double)z - f.t[2];
  // p_loc = R^T (p - t): column j of R against the offset
  xl = irr_term(irr_term(irr_term(0.0, f.R[0], dx), f.R[3], dy), f.R[6], dz);
  yl = irr_term(irr_term(irr_term(0.0, f.R[1], dx), f.R[4], dy), f.R[7], dz);
}

// Flat bin hist[ix * ny + iy] of one ray, or -1 when it is dropped (power not > 0, outside the edges, NaN / inf).
template <typename T>
OLB_IRR_HD int64_t irr_ray_bin(T x, T y, T z, T power, const IrrFrame& f, const double* xe, int32_t nx, double x_inv,
                               const double* ye, int32_t ny, double y_inv) {
  if (!(power > (T)0)) return -1;
  double xl, yl;
  irr_localize<T>(x, y, z, f, xl, yl);
  const int32_t ix = irr_bin(xl, xe, nx, x_inv);
  if (ix < 0) return -1;
  const int32_t iy = irr_bin(yl, ye, ny, y_inv);
  if (iy < 0) return -1;
  return (int64_t)ix * ny + iy;
}

}  // namespace olb
#endif  // OLB_IRRADIANCE_CUH_
