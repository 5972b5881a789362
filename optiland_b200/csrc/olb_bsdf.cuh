// olb_bsdf.cuh -- BSDF scatter of one ray (OLB_SF_BSDF; include/olb.h "BSDF scatter"): Optiland's LambertianBSDF /
// GaussianBSDF (optiland/scatter.py) with counter-based random numbers, so the draws of a ray are a pure function of
// (surface seed, ray index, call stream, attempt) on the device and in the host instantiation alike.
//
// Included after olb_math.cuh by the translation units that instantiate FEAT_BSDF kernels (olb_trace.cu and the host
// check); olb_math.cuh only declares bsdf_scatter.
#ifndef OLB_BSDF_CUH_
#define OLB_BSDF_CUH_

#if !defined(__CUDACC__)
#include <cuda_runtime.h>   // uint2 / uint4 and the __host__ __device__ qualifiers for the host instantiation
#endif
#ifndef QUALIFIERS
#define QUALIFIERS static __forceinline__ __host__ __device__   // cuRAND's Philox, compiled for host and device
#endif
#include <curand_philox4x32_x.h>

#include "olb_math.cuh"

namespace olb {

// A 53-bit uniform in [0, 1) from two 32-bit words: (hi >> 5) * 2^26 + (lo >> 6), over 2^53.
OLB_HD uint64_t bsdf_bits53(uint32_t hi, uint32_t lo) { return ((uint64_t)(hi >> 5) << 26) | (uint64_t)(lo >> 6); }

// Draw number `attempt` of ray `ray` (include/olb.h): the disk / Gaussian point (x, y) of the scatter loop.  kind and
// sigma are the surface's block values; the two uniforms are formed in fp64 and rounded to T.
template <typename T>
OLB_HD void bsdf_draw(uint64_t key, uint64_t ray, uint32_t stream, uint32_t attempt, int kind, T sigma, T& x, T& y) {
  uint4 ctr;
  ctr.x = (uint32_t)ray; ctr.y = (uint32_t)(ray >> 32); ctr.z = stream; ctr.w = attempt;
  uint2 k;
  k.x = (uint32_t)key; k.y = (uint32_t)(key >> 32);
  const uint4 w = curand_Philox4x32_10(ctr, k);
  const uint64_t a = bsdf_bits53(w.x, w.y), b = bsdf_bits53(w.z, w.w);
  const T v = (T)((double)b * 0x1p-53);
  const T theta = (T)(2.0 * M_PI) * v;
  const T c = cos(theta), s = sin(theta);
  if (kind == OLB_BSDF_GAUSSIAN) {
    // Box-Muller (get_point_gaussian): u1 in (0, 1], so log u1 is finite and rho never inf
    const T u1 = (T)((double)(a + 1) * 0x1p-53);
    const T rho = sqrt((T)-2 * log(u1));
    x = sigma * (rho * c);
    y = sigma * (rho * s);
  } else {
    // point on the unit disk (get_point_lambertian)
    const T sr = sqrt((T)((double)a * 0x1p-53));
    x = sr * c;
    y = sr * s;
  }
}

// The scatter step: (r.L, r.M, r.N) := a direction drawn about the interaction's outgoing direction in the frame of the
// geometry's UNALIGNED normal n, with the reference's operation order (scatter.py:scatter).  `bs` is the prepared block
// (olb_prep.h BS_*).  A ray that exhausts OLB_BSDF_MAX_ATTEMPTS leaves with a NaN direction.
template <typename T>
OLB_HD void bsdf_scatter(Ray<T>& r, const T* bs, T nx, T ny, T nz, int& status) {
  const int kind = (int)bs[BS_KIND];
  const T sigma = bs[BS_SIGMA];
  uint64_t key = 0;
  for (int q = 0; q < 4; ++q) key |= (uint64_t)(uint32_t)bs[BS_KEY + q] << (16 * q);
  const T n[3] = {nx, ny, nz};
  const bool xref = r.L < (T)0.999;                       // arbitrary_vector: (1, 0, 0), else (0, 1, 0)
  const T arb[3] = {xref ? (T)1 : (T)0, xref ? (T)0 : (T)1, (T)0};
  T a[3], b[3];
  o_cross(n, arb, a);
  const T nrm = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
  a[0] = a[0] / nrm; a[1] = a[1] / nrm; a[2] = a[2] / nrm;   // n parallel to arb: 0 / 0, a NaN direction
  o_cross(n, a, b);
  const T ra = r.L * a[0] + r.M * a[1] + r.N * a[2];
  const T rb = r.L * b[0] + r.M * b[1] + r.N * b[2];
  T sx = 0, sy = 0, rad = 0;
  uint32_t attempt = 0;
  for (; attempt < (uint32_t)OLB_BSDF_MAX_ATTEMPTS; ++attempt) {
    T x, y;
    bsdf_draw<T>(key, r.id, r.stream, attempt, kind, sigma, x, y);
    sx = ra + x;
    sy = rb + y;
    rad = (T)1 - sx * sx - sy * sy;
    if (!(rad < 0)) break;                                 // accepted; a NaN radicand ends the loop as well
  }
  if (attempt == (uint32_t)OLB_BSDF_MAX_ATTEMPTS) {
    status |= OLB_ST_BSDF_ATTEMPTS;
    sx = sy = rad = (T)NAN;
  }
  const T sz = sqrt(rad);
  r.L = sx * a[0] + sy * b[0] + sz * n[0];
  r.M = sx * a[1] + sy * b[1] + sz * n[1];
  r.N = sx * a[2] + sy * b[2] + sz * n[2];
}

}  // namespace olb
#endif  // OLB_BSDF_CUH_
