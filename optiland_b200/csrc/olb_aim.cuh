// olb_aim.cuh -- per-ray ray-aiming solve (include/olb.h: OlbAimCall).
//
// One solve of Optiland's IterativeRayAimer.aim_rays (optiland/rays/ray_aiming/iterative.py:60-281) from a given
// guess, for ONE ray: the reference iterates on the whole batch, but a ray's iterates never depend on another
// ray's -- a converged ray keeps its parameters (re-tracing it reproduces its error bit for bit), a non-converged ray
// takes its own Newton step and its own Broyden update, a NaN ray never converges.  So the batch loop becomes a
// per-thread loop with no host round trip in between; what the reference raises becomes a status bit.
//
// The step is the reference's, in the element type and in its operation order: products that the reference adds
// are formed by o_mul_nc (no fused multiply-add), and the divisions are IEEE divisions (not o_div's fp32 reciprocal).
// __host__ __device__: tests/hostcheck/hostcheck_aim.cpp instantiates the same code on the CPU.
#ifndef OLB_AIM_CUH_
#define OLB_AIM_CUH_

#include "olb_math.cuh"

namespace olb {

// Kernel variant of an aim table (the trace kernel's instantiations, unpolarized): closed form, general, or the
// phase / grating / grid-sag / polygon superset.  -1: not built (BSDF scatter; Fresnel / Jones coatings need
// polarized rays, which the aimer never traces; Forbes Q-2D surfaces, whose code only the trace kernels carry).
enum { AIM_CLOSED_FORM = 0, AIM_GENERAL = 1, AIM_SUPERSET = 2 };
constexpr uint32_t AIM_FEAT_GENERAL = FEAT_ROT | FEAT_NEWTON | FEAT_EXTRA | FEAT_FREEFORM;
constexpr uint32_t AIM_FEAT_SUPERSET = AIM_FEAT_GENERAL | FEAT_PHASE | FEAT_GRATING | FEAT_GRID | FEAT_POLYGON;

inline int aim_variant(uint32_t features) {
  if (features & (FEAT_BSDF | FEAT_POL | FEAT_JONES | FEAT_Q2D)) return -1;
  if (features & (FEAT_PHASE | FEAT_GRATING | FEAT_GRID | FEAT_POLYGON)) return AIM_SUPERSET;
  if ((features & ~uint32_t(FEAT_ROT)) == 0) return AIM_CLOSED_FORM;
  return AIM_GENERAL;
}

// Trace one launch state through surfaces [first, last) (IterativeRayAimer._trace_subset: intensity 1, OPD 0) and
// return its intercept in the LOCAL frame of surface last - 1 -- what _get_local_stop_coords computes by localizing
// the global record again.  The caller guarantees that surface last - 1 is not the object surface.
template <typename T, uint32_t FEAT>
OLB_HD void aim_trace(const PrepSurface<T>* surf, const T* pool, int first, int last, T x, T y, T z, T L, T M, T N,
                      int widx, T& lx, T& ly, int& status) {
  Ray<T> r{};
  r.x = x; r.y = y; r.z = z; r.L = L; r.M = M; r.N = N;
  r.i = (T)1; r.opd = (T)0; r.opd_lo = (T)0; r.widx = widx;
  bool have_frame = false;
  for (int s = first; s < last; ++s) {
    if (surf[s].kind == OLB_GEOM_NOOP) continue;
    surface_step<T, FEAT>(r, surf[s], pool, !have_frame, status);
    have_frame = true;
  }
  lx = r.x; ly = r.y;
}

// The solve for one ray.  (x, y, L, M) are updated in place: (x, y) for an infinite object, (L, M) otherwise, with
// N left as it is (the reference does not renormalise it).  tx, ty: the target on the stop, Px r_stop and Py r_stop.
// Returns the OLB_ST_* bits: OLB_ST_AIM_NAN_START (initial x error NaN, iterative.py:141-145), OLB_ST_AIM_UNCONVERGED
// (not converged after max_iter steps, :278-279) and the trace's own bits (Zernike / Chebyshev range).
template <typename T, uint32_t FEAT>
OLB_HD int aim_ray(const PrepSurface<T>* surf, const T* pool, int first, int last, T& x, T& y, T z, T& L, T& M, T N,
                   int widx, T tx, T ty, T Jf, T tol_sq, int max_iter, bool infinite) {
  int status = 0;
  T ex, ey;
  aim_trace<T, FEAT>(surf, pool, first, last, x, y, z, L, M, N, widx, ex, ey, status);
  ex = ex - tx; ey = ey - ty;
  if (ex != ex) return status | OLB_ST_AIM_NAN_START;
  T J11 = Jf, J12 = (T)0, J21 = (T)0, J22 = Jf;      // J = diag(J_factor)
  const T det_floor = (T)1e-12, nsq_floor = (T)1e-20;
  for (int it = 0; it < max_iter; ++it) {
    if (o_mul_nc(ex, ex) + o_mul_nc(ey, ey) < tol_sq) return status;    // (NaN: never converged)
    T det = o_mul_nc(J11, J22) - o_mul_nc(J12, J21);
    if (o_abs(det) < det_floor) det = det_floor;
    const T dp1 = -(o_mul_nc(J22, ex) + o_mul_nc(-J12, ey)) / det;
    const T dp2 = -(o_mul_nc(-J21, ex) + o_mul_nc(J11, ey)) / det;
    if (infinite) { x = x + dp1; y = y + dp2; }
    else { L = L + dp1; M = M + dp2; }
    T exn, eyn;
    aim_trace<T, FEAT>(surf, pool, first, last, x, y, z, L, M, N, widx, exn, eyn, status);
    exn = exn - tx; eyn = eyn - ty;
    // Broyden rank-1 update with the OLD J: J += (dE - J dp) dp^T / max(|dp|^2, 1e-20)
    const T Rx = (exn - ex) - (o_mul_nc(J11, dp1) + o_mul_nc(J12, dp2));
    const T Ry = (eyn - ey) - (o_mul_nc(J21, dp1) + o_mul_nc(J22, dp2));
    T nsq = o_mul_nc(dp1, dp1) + o_mul_nc(dp2, dp2);
    if (!(nsq != nsq) && !(nsq > nsq_floor)) nsq = nsq_floor;           // torch.maximum: NaN propagates
    J11 = J11 + o_mul_nc(Rx, dp1) / nsq;
    J12 = J12 + o_mul_nc(Rx, dp2) / nsq;
    J21 = J21 + o_mul_nc(Ry, dp1) / nsq;
    J22 = J22 + o_mul_nc(Ry, dp2) / nsq;
    ex = exn; ey = eyn;
  }
  if (!(o_mul_nc(ex, ex) + o_mul_nc(ey, ey) < tol_sq)) status |= OLB_ST_AIM_UNCONVERGED;
  return status;
}

// Wavelength index of a ray in the table's wavelength list (-1: not in it -> NaN, as in the trace kernel).
template <typename T>
OLB_HD int aim_widx(const T* wl, int n_wl, T w) {
  int idx = -1;
  for (int j = 0; j < n_wl; ++j)
    if (w == wl[j]) idx = j;
  return idx;
}

}  // namespace olb

#endif  // OLB_AIM_CUH_
