// olb_math.cuh -- per-ray arithmetic of the real-ray trace hot path.
//
// One templated function, `surface_step`, does for ONE ray at ONE surface what the
// reference does with ~190 element-wise array ops (SURVEY.md section 1):
//   localize -> distance -> propagate + OPD (+ absorption) -> clip -> normal ->
//   refract / reflect -> coating
// and leaves the ray in the surface's LOCAL frame (the caller globalizes for the
// record).  Reference: optiland/surfaces/standard_surface.py:232-248 and the
// functions cited at each block below.
//
// The functions are __host__ __device__ so that the very same arithmetic can be
// instantiated on the CPU by tests/hostcheck (test infrastructure; never shipped in
// libolb.so) and checked against the oracle in the GPU-less build container.
#ifndef OLB_MATH_CUH_
#define OLB_MATH_CUH_

#include <math.h>
#include <stdint.h>

#include "olb_prep.h"

#if defined(__CUDACC__)
#define OLB_HD __host__ __device__ __forceinline__
#ifdef OLB_NEWTON_CALL   // tuning knob: Newton solve as an out-of-line call (slower: spills around the call)
#define OLB_HD_CALL __host__ __device__ __noinline__
#else
#define OLB_HD_CALL __host__ __device__ __forceinline__
#endif
#else
#define OLB_HD inline
#define OLB_HD_CALL inline
#endif

namespace olb {

// ---- scalar helpers: IEEE for double; for float on the device the single-instruction MUFU
// forms (<= 2 ulp, flush-to-zero: no denormal fix-up code around every rcp / sqrt) ----
OLB_HD double o_sqrt(double v) { return sqrt(v); }
OLB_HD double o_div(double a, double b) { return a / b; }
OLB_HD double o_rcp(double a) { return 1.0 / a; }
OLB_HD double o_rsqrt(double a) { return 1.0 / sqrt(a); }
OLB_HD double o_abs(double a) { return fabs(a); }
OLB_HD double o_exp(double a) { return exp(a); }
OLB_HD double o_fma(double a, double b, double c) { return fma(a, b, c); }
OLB_HD float o_abs(float a) { return fabsf(a); }
OLB_HD float o_fma(float a, float b, float c) { return fmaf(a, b, c); }
#if defined(__CUDA_ARCH__)
OLB_HD float o_sqrt(float v) { float r; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v)); return r; }
OLB_HD float o_rcp(float v) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v)); return r; }
OLB_HD float o_rsqrt(float v) { float r; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v)); return r; }
OLB_HD float o_div(float a, float b) { return a * o_rcp(b); }
// exp(a) = 2^(a log2 e): one FMUL + MUFU.EX2 (flush-to-zero; attenuation factors are O(1))
OLB_HD float o_exp(float a) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a * 1.4426950408889634f)); return r; }
#else
OLB_HD float o_sqrt(float v) { return sqrtf(v); }
OLB_HD float o_rcp(float v) { return 1.0f / v; }
OLB_HD float o_rsqrt(float v) { return 1.0f / sqrtf(v); }
OLB_HD float o_div(float a, float b) { return a / b; }
OLB_HD float o_exp(float a) { return expf(a); }
#endif

// Product that the compiler must NOT fuse into an FMA: cross products of (nearly) parallel
// vectors rely on a*b - b*a cancelling exactly, which fma(a, b, -round(b*a)) does not.
#if defined(__CUDA_ARCH__)
OLB_HD float o_mul_nc(float a, float b) { return __fmul_rn(a, b); }
OLB_HD double o_mul_nc(double a, double b) { return __dmul_rn(a, b); }
#else
OLB_HD float o_mul_nc(float a, float b) { volatile float p = a * b; return p; }
OLB_HD double o_mul_nc(double a, double b) { volatile double p = a * b; return p; }
#endif
template <typename T>
OLB_HD void o_cross(const T* a, const T* b, T* c) {
  c[0] = o_mul_nc(a[1], b[2]) - o_mul_nc(a[2], b[1]);
  c[1] = o_mul_nc(a[2], b[0]) - o_mul_nc(a[0], b[2]);
  c[2] = o_mul_nc(a[0], b[1]) - o_mul_nc(a[1], b[0]);
}

template <typename T> struct Eps;
template <> struct Eps<float> { static constexpr float v = 1.1920929e-7f; };
template <> struct Eps<double> { static constexpr double v = 2.220446049250313e-16; };

// Ray state held in registers. Position/direction are in the CURRENT frame (global at
// entry, then the local frame of the last traced surface).
template <typename T>
struct Ray {
  T x, y, z, L, M, N, i, opd;
  T opd_lo;    // fp32 only: low word of a two-float OPD accumulator (see accumulate_opd)
  T L0, M0, N0;  // direction before the last interaction (real_rays.py:170-172)
  int widx;    // wavelength index into the media tables
  uint64_t id;      // FEAT_BSDF only: the ray's index, counter of its scatter draws (olb_bsdf.cuh)
  uint32_t stream;  //                 and the call's rng_stream
  T P[18];     // FEAT_POL only: 3x3 complex polarization matrix, P[2*(3r+c)] = Re, +1 = Im
               // (optiland/rays/polarized_rays.py:50); untouched (and optimised away) otherwise
};

// OPD accumulation: opd += |t * n1|  (standard_surface.py:244).  In fp32 the sum is
// carried as an unevaluated (hi, lo) pair (Knuth TwoSum) so that the ~190 mm optical
// path of a camera lens does not lose 0.3 lambda to 13 roundings as the reference's own
// fp32 path does (SURVEY.md section 8d "precision reality check").
OLB_HD void accumulate_opd(Ray<double>& r, double v) { r.opd += v; }
OLB_HD void accumulate_opd(Ray<float>& r, float v) {
  float s = r.opd + v;
  float bb = s - r.opd;
  float err = (r.opd - (s - bb)) + (v - bb);
  r.opd = s;
  r.opd_lo += err;
}
OLB_HD double opd_value(const Ray<double>& r) { return r.opd; }
OLB_HD float opd_value(const Ray<float>& r) { return r.opd + r.opd_lo; }
OLB_HD double opd_value_f64(const Ray<double>& r) { return r.opd; }
OLB_HD double opd_value_f64(const Ray<float>& r) { return (double)r.opd + (double)r.opd_lo; }  // both halves

// Launch state of one ray from its pupil point (include/olb.h: OlbPupilLaunch; reference:
// rays/ray_aiming/paraxial.py:85-105 on top of fields/field_types/angle.py:40-57).
template <typename T>
OLB_HD void pupil_launch(Ray<T>& r, T Px, T Py, const T* o0, const T* os, const T* t0, const T* ts, T inten,
                         T ofx = 0, T ofy = 0, T tfx = 0, T tfy = 0) {
  // (ofx, ofy, tfx, tfy): per-ray field offsets of origin and target, 0 for a single-field launch
  r.x = o_fma(os[0], Px, o0[0]) + ofx;
  r.y = o_fma(os[1], Py, o0[1]) + ofy;
  r.z = o0[2];
  T dx = (o_fma(ts[0], Px, t0[0]) + tfx) - r.x, dy = (o_fma(ts[1], Py, t0[1]) + tfy) - r.y, dz = t0[2] - r.z;
  T mag = o_sqrt(o_fma(dx, dx, o_fma(dy, dy, dz * dz)));
  const bool zero = mag < (T)1e-9;
  T inv = o_rcp(zero ? (T)1 : mag);
  r.L = zero ? (T)0 : dx * inv;
  r.M = zero ? (T)0 : dy * inv;
  r.N = zero ? (T)1 : dz * inv;
  r.i = inten;
  r.opd = 0;
}

// Wavefront epilogue (SURVEY.md 8f-2): OPD of one traced ray against a spherical reference centred on the
// chief ray's image point, and the point where the ray meets that sphere -- steps 4-5 of
// ChiefRayStrategy.compute_wavefront_data (optiland/wavefront/strategy.py:179-190) with
// SphericalReference.path_length (optiland/wavefront/reference_geometry.py:55-82) and the launch-plane tilt
// term of _correct_tilt (strategy.py:93-139).  Always evaluated in fp64: c = |p - centre|^2 - R^2 cancels
// ~R^2 against ~R^2, and the result is wanted to 1e-5 waves.
struct WavefrontRef {
  double c[3], R, n_image, tilt[2], opd_ref, inv_wl;   // inv_wl = 1 / (wavelength[um] * 1e-3) : waves per mm
};
OLB_HD void wavefront_point(double x, double y, double z, double L, double M, double N, double opd, double Px,
                            double Py, const WavefrontRef& w, double& opd_wv, double& px, double& py, double& pz) {
  const double Lr = -L, Mr = -M, Nr = -N;               // traced backwards from the image surface
  const double a = Lr * Lr + Mr * Mr + Nr * Nr;
  const double b = 2 * (Lr * (x - w.c[0]) + Mr * (y - w.c[1]) + Nr * (z - w.c[2]));
  const double c = x * x + y * y + z * z - 2 * (x * w.c[0] + y * w.c[1] + z * w.c[2]) + w.c[0] * w.c[0] +
                   w.c[1] * w.c[1] + w.c[2] * w.c[2] - w.R * w.R;
  double d = b * b - 4 * a * c;
  if (d < 0) d = 0;
  const double sq = sqrt(d);
  const double t1 = (-b - sq) / (2 * a), t2 = (-b + sq) / (2 * a);
  const double t = t1 < 0 ? t2 : t1;
  const double opd_img = w.n_image * t;
  const double o = opd - opd_img + (w.tilt[0] * Px + w.tilt[1] * Py);
  opd_wv = (w.opd_ref - o) * w.inv_wl;
  const double tt = opd_img / w.n_image;
  px = x - tt * L; py = y - tt * M; pz = z - tt * N;
}

template <typename T>
OLB_HD void apply_affine(const T* A, const T* b, bool rotated, T& x, T& y, T& z, T& L, T& M, T& N) {
  if (rotated) {
    T px = x, py = y, pz = z, dl = L, dm = M, dn = N;
    x = o_fma(A[0], px, o_fma(A[1], py, o_fma(A[2], pz, b[0])));
    y = o_fma(A[3], px, o_fma(A[4], py, o_fma(A[5], pz, b[1])));
    z = o_fma(A[6], px, o_fma(A[7], py, o_fma(A[8], pz, b[2])));
    L = o_fma(A[0], dl, o_fma(A[1], dm, A[2] * dn));
    M = o_fma(A[3], dl, o_fma(A[4], dm, A[5] * dn));
    N = o_fma(A[6], dl, o_fma(A[7], dm, A[8] * dn));
  } else {
    x += b[0]; y += b[1]; z += b[2];
  }
}

// ---- closed-form conic intersection -----------------------------------------------
// optiland/geometries/standard.py:97-148.  Same roots t1 = (-b+sqrt(d))/2a,
// t2 = (-b-sqrt(d))/2a and the same selection rule (|z1| <= |z2| -> t1, a == 0 -> -c/b),
// but evaluated with the cancellation-free pairing q = -(b/2 + sign(b) sqrt(d/4)),
// {q/a, c/q}: the reference's form loses ~3e-9 mm on a 10^4-mm telescope in fp64 and is
// unusable in fp32 there (SURVEY.md section 8d).
template <typename T>
OLB_HD T conic_distance(T x, T y, T z, T L, T M, T N, const PrepSurface<T>& S) {
  if (S.flags & PSF_RADIUS_INF) {
    T Ns = o_abs(N) > (T)1e-14 ? N : (T)1e-14;
    return -o_div(z, Ns);
  }
  const T k = S.conic, R = S.radius;
  T a = o_fma(k * N, N, o_fma(L, L, o_fma(M, M, N * N)));
  T zz = o_fma(S.kp1, z, -R);                          // (1+k) z - R
  T hb = o_fma(L, x, o_fma(M, y, N * zz));             // b / 2
  T c = o_fma(x, x, o_fma(y, y, z * (zz - R)));        // x^2 + y^2 + z((1+k) z - 2R)
  T disc = o_fma(hb, hb, -a * c);                      // d / 4
  T sq = o_sqrt(disc);
  T q = hb >= 0 ? -(hb + sq) : (sq - hb);
  T ta = o_div(q, a);
  T tb = o_div(c, q);
  T t1 = hb >= 0 ? tb : ta;                            // (-b + sqrt d) / 2a
  T t2 = hb >= 0 ? ta : tb;                            // (-b - sqrt d) / 2a
  T z1 = o_fma(t1, N, z), z2 = o_fma(t2, N, z);
  // Degenerate inputs need no extra branches: a == 0 (paraboloid hit by an axial ray) makes
  // ta = +-inf, so the comparison keeps tb = c/q = -c/b, the reference's a == 0 value
  // (standard.py:144-146); q == 0 (b = d = 0) makes tb = NaN, and since hb >= 0 then holds the
  // comparison is false and t2 = ta = 0, the reference's double root.
  return (o_abs(z1) <= o_abs(z2)) ? t1 : t2;
}

// Conic part of the sag and of the slope denominators.
//   sag   = r2 / (R (1 + sqrt(1 - (1+k) r2 / R^2)))        standard.py:80-95
//   slope = (x, y) / (R sqrt(1 - (1+k) r2 / R^2))           standard.py:163-167
template <typename T>
OLB_HD void conic_sag_slope(T r2, const PrepSurface<T>& S, T& sag, T& inv_denom) {
  T s2 = o_fma(-S.kp1 * r2, S.curv * S.curv, (T)1);
  T s = o_sqrt(s2);
  sag = o_div(r2 * S.curv, (T)1 + s);
  inv_denom = o_div(S.curv, s);
}

// Bivariate polynomial P(x, y) = sum_ij C[i*cols+j] x^i y^j with both partials (nested
// Horner).  `tri`: table is triangular (i + j <= rows - 1), skip the structural zeros.
template <typename T>
OLB_HD void poly2_eval(const T* C, int rows, int cols, bool tri, T x, T y, T& P, T& Px, T& Py) {
  P = 0; Px = 0; Py = 0;
  for (int i = rows - 1; i >= 0; --i) {
    const T* row = C + i * cols;
    const int jmax = tri ? (rows - 1 - i) : (cols - 1);
    T q = 0, qy = 0;
#pragma unroll 4
    for (int j = jmax; j >= 0; --j) {
      qy = o_fma(qy, y, q);
      q = o_fma(q, y, row[j]);
    }
    Px = o_fma(Px, x, P);
    P = o_fma(P, x, q);
    Py = o_fma(Py, x, qy);
  }
}
template <typename T>
OLB_HD T poly2_value(const T* C, int rows, int cols, bool tri, T x, T y) {
  T P = 0;
  for (int i = rows - 1; i >= 0; --i) {
    const T* row = C + i * cols;
    const int jmax = tri ? (rows - 1 - i) : (cols - 1);
    T q = 0;
#pragma unroll 4
    for (int j = jmax; j >= 0; --j) q = o_fma(q, y, row[j]);
    P = o_fma(P, x, q);
  }
  return P;
}

// Value, gradient and Hessian of a bivariate polynomial table in one nested Horner pass (backward pass only: the
// adjoint of the surface normal needs the second partials of the slope polynomial).
template <typename T>
OLB_HD void poly2_hess(const T* C, int rows, int cols, bool tri, T x, T y, T& P, T& Px, T& Py, T& Pxx, T& Pxy, T& Pyy) {
  P = 0; Px = 0; Py = 0; Pxx = 0; Pxy = 0; Pyy = 0;
  for (int i = rows - 1; i >= 0; --i) {
    const T* row = C + i * cols;
    const int jmax = tri ? (rows - 1 - i) : (cols - 1);
    T q = 0, q1 = 0, q2 = 0;
    for (int j = jmax; j >= 0; --j) {
      q2 = o_fma(q2, y, (T)2 * q1);
      q1 = o_fma(q1, y, q);
      q = o_fma(q, y, row[j]);
    }
    Pxx = o_fma(Pxx, x, (T)2 * Px);
    Px = o_fma(Px, x, P);
    P = o_fma(P, x, q);
    Pxy = o_fma(Pxy, x, Py);
    Py = o_fma(Py, x, q1);
    Pyy = o_fma(Pyy, x, q2);
  }
}

// Triangular tables of a COMPILE-TIME width W (Zernike sums: prepare_table pads the monomial table to W in {4, 8,
// 12}).  The same nested Horner as poly2_value / poly2_eval, operation for operation (padding only prepends zero
// terms), but fully unrolled: every coefficient is a load at a constant offset and every term one FMA (value) or two
// (partials), where the runtime-sized loops spent ~8 instructions per term on index arithmetic, compare and branch --
// most of the Zernike kernel's instructions.
// Row i of a W-wide table (W a multiple of 4, the table 16-byte aligned: prepare_table): the W - i leading
// coefficients with 128-bit shared-memory loads -- 12 loads for W = 8 where scalar loads need 36.
template <typename T> struct alignas(16) CoefVec { T v[16 / sizeof(T)]; };
template <typename T, int W, int I>
OLB_HD void tri_row(const T* C, T (&row)[W]) {
  constexpr int PER = 16 / (int)sizeof(T);
  constexpr int NV = (W - I + PER - 1) / PER;
#if defined(__CUDA_ARCH__)
#pragma unroll
  for (int q = 0; q < NV; ++q) {
    const CoefVec<T> v = *reinterpret_cast<const CoefVec<T>*>(C + I * W + q * PER);
#pragma unroll
    for (int k = 0; k < PER; ++k) row[q * PER + k] = v.v[k];
  }
#else
  for (int j = 0; j < NV * PER; ++j) row[j] = C[I * W + j];
#endif
}
template <typename T, int W, int I>
struct TriRows {
  static OLB_HD void value(const T* C, T x, T y, T& P) {
    T row[W];
    tri_row<T, W, I>(C, row);
    T q = 0;
#pragma unroll
    for (int j = W - 1 - I; j >= 0; --j) q = o_fma(q, y, row[j]);
    P = o_fma(P, x, q);
    if constexpr (I > 0) TriRows<T, W, I - 1>::value(C, x, y, P);
  }
  static OLB_HD void grad(const T* C, T x, T y, T& P, T& Px, T& Py) {
    T row[W];
    tri_row<T, W, I>(C, row);
    T q = 0, qy = 0;
#pragma unroll
    for (int j = W - 1 - I; j >= 0; --j) {
      qy = o_fma(qy, y, q);
      q = o_fma(q, y, row[j]);
    }
    Px = o_fma(Px, x, P);
    P = o_fma(P, x, q);
    Py = o_fma(Py, x, qy);
    if constexpr (I > 0) TriRows<T, W, I - 1>::grad(C, x, y, P, Px, Py);
  }
};
template <typename T, int W>
OLB_HD T tri_value(const T* C, T x, T y) {
  T P = 0;
  TriRows<T, W, W - 1>::value(C, x, y, P);
  return P;
}
template <typename T, int W>
OLB_HD void tri_grad(const T* C, T x, T y, T& P, T& Px, T& Py) {
  P = 0; Px = 0; Py = 0;
  TriRows<T, W, W - 1>::grad(C, x, y, P, Px, Py);
}
// warp-uniform dispatch on the table width (one case is executed per surface; the others are never fetched)
template <typename T>
OLB_HD T poly_tri_value(const T* C, int W, T x, T y) {
  switch (W) {
    case 4: return tri_value<T, 4>(C, x, y);
    case 8: return tri_value<T, 8>(C, x, y);
    case 12: return tri_value<T, 12>(C, x, y);
    default: return poly2_value(C, W, W, true, x, y);
  }
}
template <typename T>
OLB_HD void poly_tri_grad(const T* C, int W, T x, T y, T& P, T& Px, T& Py) {
  switch (W) {
    case 4: tri_grad<T, 4>(C, x, y, P, Px, Py); break;
    case 8: tri_grad<T, 8>(C, x, y, P, Px, Py); break;
    case 12: tri_grad<T, 12>(C, x, y, P, Px, Py); break;
    default: poly2_eval(C, W, W, true, x, y, P, Px, Py);
  }
}

// Sag of a Newton-family surface at (x, y).  `status` collects OLB_ST_* bits.
//   even asphere  even_asphere.py:93-109   conic + sum C_i r2^(i+1)
//   odd asphere   odd_asphere.py:86-101    conic + sum C_i r^(i+1)
//   polynomial    polynomial.py:105-121    conic + sum C_ij x^i y^j
//   Zernike       zernike.py:153-180       conic + sum c_i N_i Z_i(rho, phi), monomial form
// Biconic profile helpers (biconic.py:72-160): z_u = c u^2 / (1 + sqrt(clamp(1 - (1+k) c^2 u^2))), the
// reference clamps the radicand to 0 (sag) / 1e-14 (slope) below 1e-14.
template <typename T>
OLB_HD T biconic_profile(T u, T c, T kp1) {
  if (c == 0) return 0;
  T v = o_fma(-kp1 * c * c, u * u, (T)1);
  T rt = v < (T)1e-14 ? (T)0 : v;
  return o_div(c * u * u, (T)1 + o_sqrt(rt));
}
template <typename T>
OLB_HD T biconic_slope(T u, T c, T kp1) {
  if (c == 0) return 0;
  T v = o_fma(-kp1 * c * c, u * u, (T)1);
  T rt = v < (T)1e-14 ? (T)1e-14 : v;
  return o_div(c * u, o_sqrt(rt));
}
// Toroidal Y-Z curve (toroidal.py:87-160): conic (radicand clamped at 0 / eps) + sum alpha_i y^(2(i+1)).
template <typename T>
OLB_HD void toroidal_yz(T y, const PrepSurface<T>& S, const T* pool, T& zy, T& dzy) {
  const T c = S.curv_y, y2 = y * y;
  zy = 0; dzy = 0;
  if (c != 0) {
    T v = o_fma(-S.kp1_y * c * c, y2, (T)1);
    zy = o_div(c * y2, (T)1 + o_sqrt(v < 0 ? (T)0 : v));
    dzy = o_div(c * y, o_sqrt(v < (T)1e-14 ? (T)1e-14 : v));
  }
  const T* a = pool + S.coef_off;
  T h = 0, hd = 0;
#pragma unroll 4
  for (int i = S.n_coef - 1; i >= 0; --i) {
    h = o_fma(h, y2, a[i]);
    hd = o_fma(hd, y2, (T)(2 * (i + 1)) * a[i]);
  }
  zy = o_fma(h, y2, zy);
  dzy = o_fma(hd, y, dzy);
}

// Forbes Q (slope-orthogonal, "Q^bfs") radial surface, forbes/geometry.py:187-366.  S(x) = sum a_m Q_m(x) and
// dS/dx by the Clenshaw recurrences of qpoly.py:131-143, 185-212 on the change-of-basis coefficients b
// (prepared on the host): alpha_n = b_n + p alpha_{n+1} - alpha_{n+2}, p = 2 - 4x, S = 2 (alpha_0 + alpha_1);
// alpha'_n = p alpha'_{n+1} - alpha'_{n+2} - 4 alpha_{n+1}, dS/dx = 2 (alpha'_0 + alpha'_1).
template <typename T>
OLB_HD void forbes_q_sum(const T* b, int nc, T x, T& S, T& dS) {
  const T p = (T)2 - (T)4 * x;
  T a1 = 0, a2 = 0, d1 = 0, d2 = 0;          // alpha_{n+1}, alpha_{n+2}, alpha'_{n+1}, alpha'_{n+2}
  T a0 = 0, d0 = 0;
#pragma unroll 4
  for (int n = nc - 1; n >= 0; --n) {
    a0 = b[n] + p * a1 - a2;
    d0 = p * d1 - d2 - (T)4 * a1;
    if (n > 0) { a2 = a1; a1 = a0; d2 = d1; d1 = d0; }
  }
  if (nc > 1) { S = (T)2 * (a0 + a1); dS = (T)2 * (d0 + d1); }
  else { S = (T)2 * a0; dS = (T)2 * d0; }
}
// conic correction factor phi and d phi / d rho (geometry.py:152-181)
template <typename T>
OLB_HD void forbes_phi(T r2, const PrepSurface<T>& S, T& phi, T& dphi) {
  if (S.flags & PSF_RADIUS_INF) { phi = 1; dphi = 0; return; }
  const T c2 = S.curv * S.curv;
  T na = (T)1 - S.conic * c2 * r2, da = (T)1 - S.kp1 * c2 * r2;
  na = na > 0 ? na : (T)1e-12;
  da = da > 0 ? da : (T)1e-12;
  const T Nn = o_sqrt(na), D = o_sqrt(da);
  phi = o_div(Nn, D);
  dphi = o_div(c2 * o_sqrt(r2), Nn * D * D * D);
}
template <typename T>
OLB_HD T forbes_sag(T x, T y, const PrepSurface<T>& S, const T* pool) {
  const T r2 = o_fma(x, x, y * y);
  T zb = 0;                                              // _base_sag: radicand clamped at 0 (geometry.py:119-133)
  if (!(S.flags & PSF_RADIUS_INF)) {
    T arg = (T)1 - S.kp1 * r2 * S.curv * S.curv;
    zb = o_div(r2 * S.curv, (T)1 + o_sqrt(arg < 0 ? (T)0 : arg));
  }
  const T usq = r2 * S.inv_norm * S.inv_norm;
  if (S.n_coef == 0 || usq > (T)1) return zb;           // no terms / outside the normalisation radius: base conic
  T Sx, dS, phi, dphi;
  forbes_q_sum(pool + S.coef_off, S.n_coef, usq, Sx, dS);
  forbes_phi(r2, S, phi, dphi);
  return zb + usq * ((T)1 - usq) * phi * Sx;
}
template <typename T>
OLB_HD void forbes_slopes(T x, T y, const PrepSurface<T>& S, const T* pool, T& fx, T& fy) {
  const T eps = (T)1e-12;
  const T r2 = o_fma(x, x, y * y);
  const T rho = o_sqrt(r2 + eps * eps);                  // rho_safe (geometry.py:345)
  T df = 0;                                              // _base_sag_derivative (geometry.py:135-149)
  if (!(S.flags & PSF_RADIUS_INF) && S.curv != 0) {
    T arg = (T)1 - S.kp1 * S.curv * S.curv * r2;
    df = o_div(S.curv * rho, o_sqrt(arg > 0 ? arg : (T)1e-12));
  }
  if (S.n_coef > 0) {
    const T u = rho * S.inv_norm, usq = u * u;
    if (!(u >= (T)1)) {
      T Sx, dS, phi, dphi;
      forbes_q_sum(pool + S.coef_off, S.n_coef, usq, Sx, dS);
      forbes_phi(r2, S, phi, dphi);
      const T dpoly_drho = dS * (T)2 * u * S.inv_norm;
      const T dpref = ((T)2 * u - (T)4 * u * usq) * S.inv_norm;
      const T pre = usq - usq * usq;
      df += dpref * phi * Sx + pre * dphi * Sx + pre * phi * dpoly_drho;
    }
  }
  fx = df * o_div(x, rho);
  fy = df * o_div(y, rho);
}

// Forbes Q-2D freeform (include/olb.h "Forbes Q-2D"; forbes/geometry.py:539-672, qpoly.py:403-540), on the block
// olb_prep.h prepares (Q2_*).  One list of one m: the Clenshaw recurrence of clenshaw_q2d / clenshaw_q2d_der,
//   alpha_n = d_n + (A_n + B_n x) alpha_{n+1} - C_{n+1} alpha_{n+2},   alpha'_n = B_n alpha_{n+1} + (A_n + B_n x) alpha'_{n+1} - C_{n+1} alpha'_{n+2}
// (alpha above the top term = 0), and the sums S = alpha_0 / 2, S' = alpha'_0 / 2, each minus 2/5 of its alpha_3 for m = 1
// with more than 3 terms (q2d_sum_from_alphas).
template <typename T, bool SLOPES>
OLB_HD void q2d_list_sum(const T* d, const T* abc, int nl, bool m1, T x, T& S, T& dS) {
  T a1 = 0, a2 = 0, d1 = 0, d2 = 0, a0 = 0, d0 = 0, a3 = 0, d3 = 0;
  for (int n = nl - 1; n >= 0; --n) {
    const T k = o_fma(abc[3 * n + 1], x, abc[3 * n]);
    a0 = o_fma(k, a1, o_fma(-abc[3 * n + 2], a2, d[n]));
    if (SLOPES) d0 = o_fma(abc[3 * n + 1], a1, o_fma(k, d1, -abc[3 * n + 2] * d2));
    if (n == 3) { a3 = a0; d3 = d0; }
    a2 = a1; a1 = a0; d2 = d1; d1 = d0;
  }
  const T q = (m1 && nl > 3) ? (T)0.4 : (T)0;
  S = o_fma(-q, a3, (T)0.5 * a0);
  if (SLOPES) dS = o_fma(-q, d3, (T)0.5 * d0);
}
// All m > 0 at one point (_compute_m_gt0_components, qpoly.py:422-459), with (c1, s1) = (cos, sin) theta:
//   P = sum_m u^m (cos m theta S_a + sin m theta S_b)
//   DR = sum_m u^(m-1) (cos m theta (2 x S'_a + m S_a) + sin m theta (2 x S'_b + m S_b)),  x = u^2  (dP/du)
//   DT = sum_m m u^m (cos m theta S_b - sin m theta S_a)                                         (dP/dtheta)
// cos m theta, sin m theta by rotation from (c1, s1).
template <typename T, bool SLOPES>
OLB_HD void q2d_angular(const T* p, int M, T u, T x, T c1, T s1, T& P, T& DR, T& DT) {
  T cm = 1, sm = 0, um1 = 1;
  P = 0; DR = 0; DT = 0;
  for (int m = 1; m <= M; ++m) {
    const T cn = o_fma(cm, c1, -sm * s1);
    sm = o_fma(sm, c1, cm * s1);
    cm = cn;
    const T um = um1 * u;
    const int na = (int)p[Q2_NA], nb = (int)p[Q2_NB], N = (int)p[Q2_N];
    const T* abc = p + Q2_MHDR;
    const T* da = abc + 3 * N;
    T sa = 0, sap = 0, sb = 0, sbp = 0;
    if (na > 0) q2d_list_sum<T, SLOPES>(da, abc, na, m == 1, x, sa, sap);
    if (nb > 0) q2d_list_sum<T, SLOPES>(da + na, abc, nb, m == 1, x, sb, sbp);
    P = o_fma(um, o_fma(cm, sa, sm * sb), P);
    if (SLOPES) {
      const T mm = (T)m, tx = (T)2 * x;
      DR = o_fma(um1, o_fma(cm, o_fma(tx, sap, mm * sa), sm * o_fma(tx, sbp, mm * sb)), DR);
      DT = o_fma(mm * um, o_fma(cm, sb, -sm * sa), DT);
    }
    um1 = um;
    p = da + na + nb;
  }
}
// r^2 = x^2 + y^2 unfused and u = rho / norm_radius by division, as the reference forms them: the departure's u > 1 cut is
// a jump, and a point on the normalisation circle must fall on the reference's side of it
template <typename T>
OLB_HD T q2d_sag(T x, T y, const PrepSurface<T>& S, const T* pool) {
  const T r2 = o_mul_nc(x, x) + o_mul_nc(y, y);
  T zb = 0;                                              // _base_sag (geometry.py:117-131)
  if (!(S.flags & PSF_RADIUS_INF)) {
    T arg = (T)1 - S.kp1 * r2 * S.curv * S.curv;
    zb = o_div(r2 * S.curv, (T)1 + o_sqrt(arg < 0 ? (T)0 : arg));
  }
  const T* blk = pool + S.coef_off;
  const T u = o_div(o_sqrt(r2 + (T)1e-12), blk[Q2_NORM]);   // the sag's rho carries + 1e-12 (geometry.py:553)
  if (u > (T)1) return zb;
  const T usq = u * u;
  // theta = atan2(y, x): rho + 1e-12 >= 1e-6, so the reference's x + 1e-12 guard never applies; at x = y = 0,
  // atan2(+-0, x) is 0 or pi by the sign of x
  T c1, s1 = 0;
  const T rr = o_sqrt(r2);
  if (rr > 0) { const T inv = o_rcp(rr); c1 = x * inv; s1 = y * inv; }
  else c1 = copysign((T)1, x);
  T S0 = 0, dS0, P, DR, DT, phi, dphi;
  if (S.poly_rows > 0) forbes_q_sum(blk + Q2_HDR, S.poly_rows, usq, S0, dS0);
  q2d_angular<T, false>(blk + Q2_HDR + S.poly_rows, S.n_coef, u, usq, c1, s1, P, DR, DT);
  forbes_phi(r2, S, phi, dphi);
  return zb + phi * o_fma(usq * ((T)1 - usq), S0, P);
}
template <typename T>
OLB_HD void q2d_slopes(T x, T y, const PrepSurface<T>& S, const T* pool, T& fx, T& fy) {
  const T* blk = pool + S.coef_off;
  const T r2 = o_mul_nc(x, x) + o_mul_nc(y, y);
  const T rho = o_sqrt(r2);                              // no + 1e-12 here (geometry.py:628-633)
  if (rho < (T)1e-12) { fx = blk[Q2_VX]; fy = blk[Q2_VY]; return; }   // the vertex value (geometry.py:596-609)
  const T inv_rho = o_rcp(rho);
  const T c1 = x * inv_rho, s1 = y * inv_rho;
  T db = 0;                                              // _base_sag_derivative (geometry.py:133-149)
  if (!(S.flags & PSF_RADIUS_INF) && S.curv != 0) {
    const T arg = (T)1 - S.kp1 * S.curv * S.curv * r2;
    db = o_div(S.curv * rho, o_sqrt(arg > 0 ? arg : (T)1e-12));
  }
  T dsr = 0, dst = 0;
  const T u = o_div(rho, blk[Q2_NORM]);
  if (!(u > (T)1)) {
    const T usq = u * u;
    T S0 = 0, dS0 = 0, P, DR, DT, phi, dphi;
    if (S.poly_rows > 0) forbes_q_sum(blk + Q2_HDR, S.poly_rows, usq, S0, dS0);
    q2d_angular<T, true>(blk + Q2_HDR + S.poly_rows, S.n_coef, u, usq, c1, s1, P, DR, DT);
    forbes_phi(r2, S, phi, dphi);
    const T pre = usq - usq * usq;
    const T dpref = ((T)2 * u - (T)4 * u * usq) * S.inv_norm;
    const T dS0_drho = dS0 * (T)2 * u * S.inv_norm;
    dsr = (dpref * S0 + pre * dS0_drho) * phi + pre * S0 * dphi + dphi * P + phi * DR * S.inv_norm;
    dst = phi * DT;
  }
  const T g = db + dsr, h = dst * inv_rho;
  fx = o_fma(c1, g, -s1 * h);
  fy = o_fma(s1, g, c1 * h);
}

// FEAT: the Forbes code is compiled only into the general kernel (FEAT_EXTRA) -- inlined into the lean
// Newton kernel it slows the even-asphere systems down (registers, I-cache); a table with
// a Forbes surface is routed to the general kernel by prepare_table.
template <typename T, uint32_t FEAT = 0xffffffffu>
OLB_HD T newton_sag(T x, T y, const PrepSurface<T>& S, const T* pool, int& status) {
  if constexpr ((FEAT & FEAT_Q2D) != 0) {                 // Q-2D: only in the two kernels of Q-2D tables
    if (S.kind == OLB_GEOM_FORBES_Q2D) return q2d_sag(x, y, S, pool);
  }
  if constexpr ((FEAT & FEAT_EXTRA) != 0) {
    if (S.kind == OLB_GEOM_FORBES_QBFS) return forbes_sag(x, y, S, pool);
  }
  if (S.kind == OLB_GEOM_BICONIC) return biconic_profile(x, S.curv, S.kp1) + biconic_profile(y, S.curv_y, S.kp1_y);
  if (S.kind == OLB_GEOM_TOROIDAL) {
    T zy, dzy;
    toroidal_yz(y, S, pool, zy, dzy);
    if (!(S.r_rot - S.r_rot == 0)) return zy;           // infinite radius of rotation: a cylinder
    T d = S.r_rot - zy;
    T term = o_fma(d, d, -x * x);
    if (term < 0) return (T)NAN;
    T sg = d > 0 ? (T)1 : (d < 0 ? (T)-1 : (T)0);
    return zy + (d - sg * o_sqrt(term));               // toroidal.py:176-186
  }
  T r2 = o_fma(x, x, y * y);
  T sag, inv_denom;
  conic_sag_slope(r2, S, sag, inv_denom);
  if (S.kind == OLB_GEOM_EVEN_ASPHERE) {
    const T* c = pool + S.coef_off;
    T h = 0;
    for (int i = S.n_coef - 1; i >= 0; --i) h = o_fma(h, r2, c[i]);
    sag = o_fma(h, r2, sag);
  } else if (S.kind == OLB_GEOM_ODD_ASPHERE) {
    const T* c = pool + S.coef_off;
    T r = o_sqrt(r2), h = 0;
    for (int i = S.n_coef - 1; i >= 0; --i) h = o_fma(h, r, c[i]);
    sag = o_fma(h, r, sag);
  } else {
    T xn = x * S.inv_norm, yn = y * S.inv_norm_y;
    if (o_abs(xn) > (T)1 || o_abs(yn) > (T)1) {
      if (S.kind == OLB_GEOM_ZERNIKE) status |= OLB_ST_ZERNIKE_RANGE;
      if (S.kind == OLB_GEOM_CHEBYSHEV) status |= OLB_ST_CHEBYSHEV_RANGE;
    }
    if (S.flags & PSF_POLY_TRI) sag += poly_tri_value(pool + S.coef_off, S.poly_rows, xn, yn);
    else sag += poly2_value(pool + S.coef_off, S.poly_rows, S.poly_cols, false, xn, yn);
  }
  return sag;
}

// Slopes (dz/dx, dz/dy) of a Newton-family surface: the un-normalised (dfdx, dfdy) of
// even_asphere.py:111-140, odd_asphere.py:103-142, polynomial.py:123-155,
// zernike.py:182-252 (Zernike: derivative WITHOUT N_nm and exactly zero at rho == 0,
// reproducing the reference's eps-regularised chain rule).
template <typename T, uint32_t FEAT = 0xffffffffu>
OLB_HD void newton_slopes(T x, T y, const PrepSurface<T>& S, const T* pool, T& fx, T& fy) {
  if constexpr ((FEAT & FEAT_Q2D) != 0) {
    if (S.kind == OLB_GEOM_FORBES_Q2D) { q2d_slopes(x, y, S, pool, fx, fy); return; }
  }
  if constexpr ((FEAT & FEAT_EXTRA) != 0) {
    if (S.kind == OLB_GEOM_FORBES_QBFS) { forbes_slopes(x, y, S, pool, fx, fy); return; }
  }
  if (S.kind == OLB_GEOM_BICONIC) {                     // biconic.py:107-160
    fx = biconic_slope(x, S.curv, S.kp1);
    fy = biconic_slope(y, S.curv_y, S.kp1_y);
    return;
  }
  if (S.kind == OLB_GEOM_TOROIDAL) {                    // toroidal.py:188-232
    T zy, dzy;
    toroidal_yz(y, S, pool, zy, dzy);
    if (!(S.r_rot - S.r_rot == 0)) { fx = 0; fy = dzy; return; }
    T d = S.r_rot - zy;
    T term = o_fma(d, d, -x * x);
    if (!(term >= 0)) { fx = 0; fy = 0; return; }       // outside the torus: normal (0, 0, -1)
    T sq = o_sqrt(term);
    if (o_abs(sq) < (T)1e-14) sq = (T)1e-14;
    T sr = S.r_rot > 0 ? (T)1 : (T)-1;
    fx = o_div(sr * x, sq);
    fy = o_div(sr * d * dzy, sq);
    return;
  }
  T r2 = o_fma(x, x, y * y);
  T sag, g;
  conic_sag_slope(r2, S, sag, g);
  if (S.kind == OLB_GEOM_EVEN_ASPHERE) {
    const T* d = pool + S.poly_d_off;       // 2(i+1) C_i, prepared on the host
    T h = 0;
    for (int i = S.n_coef - 1; i >= 0; --i) h = o_fma(h, r2, d[i]);
    g += h;
    fx = x * g; fy = y * g;
  } else if (S.kind == OLB_GEOM_ODD_ASPHERE) {
    const T* d = pool + S.poly_d_off;       // (i+1) C_i, prepared on the host
    T r = o_sqrt(r2), h = 0;
    for (int i = S.n_coef - 1; i >= 0; --i) h = o_fma(h, r, d[i]);
    // terms (i+1) x C_i r^(i-1); non-finite terms are zeroed by the reference (r == 0)
    T hr = r > 0 ? o_div(h, r) : (T)0;
    g += hr;
    fx = x * g; fy = y * g;
  } else {
    T xn = x * S.inv_norm, yn = y * S.inv_norm_y;
    T P, Px, Py;
    if (S.flags & PSF_POLY_TRI) poly_tri_grad(pool + S.poly_d_off, S.poly_rows, xn, yn, P, Px, Py);
    else poly2_eval(pool + S.poly_d_off, S.poly_rows, S.poly_cols, false, xn, yn, P, Px, Py);
    if (S.kind == OLB_GEOM_ZERNIKE) {
      // The reference forms dZ/dx = A drho/dx + B dphi/dx with REGULARISED chain-rule factors
      //   drho/dx = xn / (R (rho + eps)),  dphi/dx = -yn / (R (rho^2 + eps)),  eps = 1e-14
      // (zernike.py:206-231).  With A = (xn Dx + yn Dy)/rho and B = xn Dy - yn Dx recovered from
      // the exact partials (Dx, Dy) this damps the slope by a = rho/(rho+eps), b = rho^2/(rho^2+eps)
      // -- 0.25 % at rho = 2e-6, exactly zero on the axis.  Reproduced, not fixed.
      const T eps = (T)1e-14;
      T rho2 = o_fma(xn, xn, yn * yn);
      if (rho2 == 0) { Px = 0; Py = 0; }
      else {
        T rho = o_sqrt(rho2);
        T a_ = o_div(rho, rho + eps), b_ = o_div(rho2, rho2 + eps), inv = o_rcp(rho2);
        T xx = xn * xn, yy = yn * yn, xy = xn * yn * (a_ - b_);
        T Dx = Px, Dy = Py;
        Px = o_fma(Dx, o_fma(a_, xx, b_ * yy), Dy * xy) * inv;
        Py = o_fma(Dy, o_fma(a_, yy, b_ * xx), Dx * xy) * inv;
      }
    }
    // Chebyshev quirk (reproduced, not fixed): the reference adds T_i'(x/norm_x) T_j(y/norm_y) to dz/dx
    // WITHOUT the chain-rule factor 1/norm_x (chebyshev.py:171-181, :206-228)
    const bool cheb = S.kind == OLB_GEOM_CHEBYSHEV;
    fx = o_fma(x, g, cheb ? Px : Px * S.inv_norm);
    fy = o_fma(y, g, cheb ? Py : Py * S.inv_norm_y);
  }
}

// Newton-Raphson refinement of t (newton_raphson.py:119-168).  The reference stops
// when max over ALL rays |f| < tol; a kernel cannot see all rays, so each ray iterates
// until its own |f| < tol and then takes ONE more step, which by quadratic convergence
// leaves a residual ~tol^2: every ray ends at least as converged as in the reference,
// and the two differ by at most the reference's own stopping residual (< tol).
// Rounding noise: the tolerance is floored at 8 eps (|z| + |sag|), and the loop also
// stops as soon as a step fails to halve |f| (quadratic convergence has ended: the
// iterate sits on the noise floor of f, which for fp32 polynomial sags lies above the
// floor estimate) keeping the better of the last two iterates -- so fp32 cannot spin
// to max_iter.
// A step that fails to halve |f| ends the iteration only NEAR the surface: |f| within 1024x the rounding noise of
// f = sag - (z + t N) itself, 8 eps (|z| + |t| + |sag|) -- the OPERANDS' magnitudes, not the result's: a ray that lands
// next to the vertex has z + t N ~ 0 with the absolute noise of |z| and |t| (fp32: ~1e-6 mm), and must still count as
// stalled on the noise floor instead of spinning to max_iter.  Far from the surface the ray is not converging at all -- it
// misses the surface, or Newton is wandering -- and the reference keeps stepping until max_iter or until an iterate leaves
// the sag's domain (NaN from then on, newton_raphson.py:137-168); so does this loop, which gives such rays the reference's
// NaN / finite pattern instead of a "best iterate" that is no intersection.
template <typename T> OLB_HD T newton_wander_bound(T z, T t, T sag) {
  return (T)1024 * (T)8 * Eps<T>::v * (o_abs(z) + o_abs(t) + o_abs(sag));
}

// Sag and slopes at the same point (one Newton iteration needs both).  Even / odd aspheres share the conic
// square root and r^2 between the two (returns with fx, fy set); for the other families only the sag is
// evaluated here and newton_distance calls newton_slopes once the convergence test has passed.
template <typename T, uint32_t FEAT = 0xffffffffu>
OLB_HD T newton_sag_slopes(T x, T y, const PrepSurface<T>& S, const T* pool, T& fx, T& fy, int& status) {
  if (S.kind == OLB_GEOM_EVEN_ASPHERE || S.kind == OLB_GEOM_ODD_ASPHERE) {
    const T r2 = o_fma(x, x, y * y);
    T sag, g;
    conic_sag_slope(r2, S, sag, g);
    const T* c = pool + S.coef_off;
    const T* d = pool + S.poly_d_off;
    T h = 0, hd = 0;
    if (S.kind == OLB_GEOM_EVEN_ASPHERE) {
#pragma unroll 4
      for (int i = S.n_coef - 1; i >= 0; --i) { h = o_fma(h, r2, c[i]); hd = o_fma(hd, r2, d[i]); }
      sag = o_fma(h, r2, sag);
      g += hd;
    } else {
      const T r = o_sqrt(r2);
#pragma unroll 4
      for (int i = S.n_coef - 1; i >= 0; --i) { h = o_fma(h, r, c[i]); hd = o_fma(hd, r, d[i]); }
      sag = o_fma(h, r, sag);
      g += r > 0 ? o_div(hd, r) : (T)0;
    }
    fx = x * g; fy = y * g;
    return sag;
  }
  fx = 0; fy = 0;                       // (not an asphere: never reached from newton_distance<.., ASPH = true>)
  return newton_sag<T, FEAT>(x, y, S, pool, status);
}

// ASPH: the surface is an even / odd asphere (compile-time, so that each family's loop carries only its own code)
template <typename T, uint32_t FEAT = 0xffffffffu, bool ASPH = false>
OLB_HD T newton_distance(T x, T y, T z, T L, T M, T N, const PrepSurface<T>& S, const T* pool, int& status) {
  T t = conic_distance(x, y, z, L, M, N, S);
  T t_prev = t, f_prev = (T)INFINITY;
  constexpr bool asphere = ASPH;
  for (int it = 0; it < S.max_iter; ++it) {
    T xi = o_fma(t, L, x), yi = o_fma(t, M, y), zi = o_fma(t, N, z);
    T fx = 0, fy = 0;
    T sag;
    if constexpr (ASPH) sag = newton_sag_slopes<T, FEAT>(xi, yi, S, pool, fx, fy, status);
    else sag = newton_sag<T, FEAT>(xi, yi, S, pool, status);
    T f = sag - zi;
    T af = o_abs(f);
    if (!(af == af)) { t = f; break; }  // sag undefined at this iterate (outside the surface's domain): the reference's
                                        // t -= f / f' turns NaN there and stays NaN to max_iter -- so does the distance
    T tol = S.tol;
    T floor_ = (T)8 * Eps<T>::v * (o_abs(zi) + o_abs(sag));
    if (floor_ > tol) tol = floor_;
    const bool conv = af < tol;
    if (!conv && !(af < (T)0.5 * f_prev) && !(af > newton_wander_bound<T>(z, t, sag))) {  // stalled on the noise floor
      if (!(af < f_prev)) t = t_prev;
      break;
    }
    if (!asphere) newton_slopes<T, FEAT>(xi, yi, S, pool, fx, fy);
    // f'(t) = fx L + fy M - N  with fx = -nx/nz = dz/dx  (newton_raphson.py:155-161)
    T df = o_fma(fx, L, o_fma(fy, M, -N));
    T dfs = o_abs(df) > (T)1e-14 ? df : (T)1e-14;
    t_prev = t; f_prev = af;
    t -= o_div(f, dfs);
    if (conv) break;  // that was the polishing step
  }
  return t;
}

// The whole Newton-family intersection: distance + slopes at the hit point.  Inlined, the Newton-capable
// kernels are 6-12 k SASS instructions; compiling this as ONE out-of-line function (-DOLB_NEWTON_CALL)
// shrinks them by 30 % but the spills around the call cost more than the I-cache misses saved
// overall), so it stays inlined.
template <typename T> struct NewtonHit { T t, fx, fy; int status; };

// The generic families (polynomial / Zernike / Chebyshev / biconic / toroidal / Forbes): the SAME iteration as
// newton_distance followed by the slopes at the hit point, arranged so that the kernel holds ONE copy of the sag code
// and ONE copy of the slope code (the unrolled polynomial evaluators are large): every exit of the loop -- converged
// and polished, stalled on the noise floor (possibly stepping back to the previous iterate), NaN, max_iter -- leaves
// through the slope evaluation at the final t.
template <typename T, uint32_t FEAT>
OLB_HD NewtonHit<T> newton_hit_generic(T x, T y, T z, T L, T M, T N, const PrepSurface<T>& S, const T* pool) {
  NewtonHit<T> h;
  h.status = 0;
  T t = conic_distance(x, y, z, L, M, N, S);
  T t_prev = t, f_prev = (T)INFINITY;
  bool final_pass = S.max_iter <= 0;
  int it = 0;
  T fx = 0, fy = 0;
  // Zernike surfaces ITERATE with the exact partials of the sag polynomial, obtained in the same pass as its value.
  // The reference iterates with its own slope function, whose Zernike part omits the normalisation constants
  // (zernike/base.py:104-136) -- an inexact f' that makes its Newton iteration converge only linearly (~4
  // evaluations where 2 suffice).  The fixed point f(t) = 0 does not depend on the slope used to reach it, so the
  // intersection is the same to within the stopping tolerance; the NORMAL at the hit point still comes from the
  // reference's slope function (newton_slopes, below).
  const bool zern = S.kind == OLB_GEOM_ZERNIKE && (S.flags & PSF_POLY_TRI) != 0;
  for (;;) {
    const T xi = o_fma(t, L, x), yi = o_fma(t, M, y);
    T f = 0, af = 0;
    bool conv = false;
    if (!final_pass) {
      const T zi = o_fma(t, N, z);
      T sag;
      if (zern) {
        T g, P, Px, Py;
        conic_sag_slope(o_fma(xi, xi, yi * yi), S, sag, g);
        const T xn = xi * S.inv_norm, yn = yi * S.inv_norm_y;
        if (o_abs(xn) > (T)1 || o_abs(yn) > (T)1) h.status |= OLB_ST_ZERNIKE_RANGE;
        poly_tri_grad(pool + S.coef_off, S.poly_rows, xn, yn, P, Px, Py);
        sag += P;
        fx = o_fma(xi, g, Px * S.inv_norm);
        fy = o_fma(yi, g, Py * S.inv_norm_y);
      } else {
        sag = newton_sag<T, FEAT>(xi, yi, S, pool, h.status);
      }
      f = sag - zi;
      af = o_abs(f);
      if (!(af == af)) {
        final_pass = true;                       // sag undefined at this iterate: the reference's t -= f / f' turns NaN
        t = f;                                   // there and stays NaN to max_iter -- so does the distance returned here
      } else {
        T tol = S.tol;
        const T floor_ = (T)8 * Eps<T>::v * (o_abs(zi) + o_abs(sag));
        if (floor_ > tol) tol = floor_;
        conv = af < tol;
        if (!conv && !(af < (T)0.5 * f_prev) && !(af > newton_wander_bound<T>(z, t, sag))) {  // stalled on the noise floor
          final_pass = true;
          if (!(af < f_prev)) { t = t_prev; continue; }   // keep the better iterate: slopes there
        }
      }
    }
    if (final_pass || !zern) newton_slopes<T, FEAT>(xi, yi, S, pool, fx, fy);
    if (final_pass) break;
    // f'(t) = fx L + fy M - N  with fx = -nx/nz = dz/dx  (newton_raphson.py:155-161)
    const T df = o_fma(fx, L, o_fma(fy, M, -N));
    const T dfs = o_abs(df) > (T)1e-14 ? df : (T)1e-14;
    t_prev = t; f_prev = af;
    t -= o_div(f, dfs);
    ++it;
    if (conv || it >= S.max_iter) final_pass = true;   // conv: that was the polishing step
  }
  h.t = t; h.fx = fx; h.fy = fy;
  return h;
}

template <typename T, uint32_t FEAT = 0xffffffffu, bool ASPH = false>
OLB_HD_CALL NewtonHit<T> newton_hit(T x, T y, T z, T L, T M, T N, const PrepSurface<T>* S, const T* pool) {
  if constexpr (!ASPH) {
    return newton_hit_generic<T, FEAT>(x, y, z, L, M, N, *S, pool);
  } else {
    NewtonHit<T> h;
    h.status = 0;
    h.t = newton_distance<T, FEAT, ASPH>(x, y, z, L, M, N, *S, pool, h.status);
    (void)newton_sag_slopes<T, FEAT>(o_fma(h.t, L, x), o_fma(h.t, M, y), *S, pool, h.fx, h.fy, h.status);
    return h;
  }
}

// ---- grid sag (GridSagGeometry, grid_sag.py:60-140; include/olb.h "Grid sag") ----------------------------------
// Prepared block at S.coef_off: x[nx], y[ny], sag[ny][nx] with nx = S.poly_cols, ny = S.poly_rows.

// searchsorted(c, p, side="right") - 1 clamped to [0, n - 2]: the number of nodes <= p, minus one (a NaN p counts none)
template <typename T>
OLB_HD int grid_cell(const T* c, int n, T p) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (c[mid] <= p) lo = mid + 1;
    else hi = mid;
  }
  const int i = lo - 1;
  return i < 0 ? 0 : (i > n - 2 ? n - 2 : i);
}

// Bilinear sag and slopes at (px, py), the reference's expressions term by term (grid_sag.py:60-100): the sag is NaN
// outside the grid, the slopes are extrapolated from the clamped cell.  sxy (nullable): the cell's mixed derivative.
template <typename T>
OLB_HD T grid_eval(const PrepSurface<T>& S, const T* pool, T px, T py, T& sx, T& sy, T* sxy = nullptr) {
  const int nx = S.poly_cols, ny = S.poly_rows;
  const T* gx = pool + S.coef_off;
  const T* gy = gx + nx;
  const int i = grid_cell(gx, nx, px), j = grid_cell(gy, ny, py);
  const T* z1 = gy + ny + j * nx + i;
  const T z11 = z1[0], z12 = z1[1], z21 = z1[nx], z22 = z1[nx + 1];
  const T dx = gx[i + 1] - gx[i], dy = gy[j + 1] - gy[j];
  const T tx = o_div(px - gx[i], dx), ty = o_div(py - gy[j], dy);
  const T ux = (T)1 - tx, uy = (T)1 - ty;
  sx = o_div((z12 - z11) * uy + (z22 - z21) * ty, dx);
  sy = o_div((z21 - z11) * ux + (z22 - z12) * tx, dy);
  if (sxy) *sxy = o_div((z22 - z21) - (z12 - z11), dx * dy);
  const bool out = px < gx[0] || px > gx[nx - 1] || py < gy[0] || py > gy[ny - 1];
  return out ? (T)NAN : (z11 * ux + z12 * tx) * uy + (z21 * ux + z22 * tx) * ty;
}

// Intersection (GridSagGeometry.distance, grid_sag.py:108-140) and the slopes at the intercept.  Newton from t = 0;
// each ray stops on its own |dt| < tol and takes one polishing step (include/olb.h explains why that agrees with the
// reference's stop on the largest |dt| of all rays).  The tolerance is floored at the rounding noise of t, so that fp32
// cannot spin to max_iter.  One copy of the interpolation serves the loop and the final out-of-grid test, which makes
// t and the slopes NaN.
template <typename T>
OLB_HD NewtonHit<T> grid_hit(T x, T y, T z, T L, T M, T N, const PrepSurface<T>& S, const T* pool) {
  NewtonHit<T> h;
  h.status = 0;
  T t = 0, sx = 0, sy = 0;
  int it = 0;
  bool polish = false, final_pass = S.max_iter <= 0;
  for (;;) {
    const T sag = grid_eval(S, pool, o_fma(t, L, x), o_fma(t, M, y), sx, sy);
    if (final_pass) {
      if (!(sag == sag)) { t = (T)NAN; sx = t; sy = t; }
      break;
    }
    const T zi = o_fma(t, N, z);
    const T dt = -o_div(sag - zi, o_fma(sx, L, o_fma(sy, M, -N)));
    t += dt;
    ++it;
    T tol = S.tol;
    const T floor_ = (T)8 * Eps<T>::v * (o_abs(t) + o_abs(zi));
    if (floor_ > tol) tol = floor_;
    if (polish || it >= S.max_iter || !(t == t)) final_pass = true;   // (a NaN iterate stays NaN in the reference)
    else if (o_abs(dt) < tol) polish = true;
  }
  h.t = t; h.fx = sx; h.fy = sy;
  return h;
}

// OLB_AP_POLYGON (include/olb.h; prepared form: olb_prep.h PG_*): the even-odd crossing count of the reference's torch
// backend over the edge records of the point's y-bucket.  x_int = vx + slope * (py - vy) with the product rounded
// before the sum, as the reference's separate array operations round it.
template <typename T>
OLB_HD bool polygon_inside(const T* pg, T x, T y) {
  const T ymin = pg[PG_YMIN];
  if (!(y >= ymin && y < pg[PG_YMAX])) return false;   // no edge has cond there (NaN included)
  const T* start = pg + (int)pg[PG_OFF];
  const int nb = (int)pg[PG_NB];
  const int b = polygon_bucket(y, ymin, pg[PG_SCALE], nb);
  const T* rec = start + ((nb + 1 + 3) & ~3);
  const int e1 = (int)start[b + 1];
  bool odd = false;
  for (int e = (int)start[b]; e < e1; ++e) {
    const T* r = rec + PG_REC * e;
    const T vy = r[1];
    const bool cond = (vy > y) != (r[2] > y);
    const T x_int = r[0] + o_mul_nc(r[3], y - vy);
    odd ^= cond && (x < x_int);
  }
  return odd;
}

// Aperture program (postfix) -> inside?   physical_apertures/*.py, see include/olb.h.  POLYGON compiles the
// polygon instruction in (FEAT_POLYGON kernels and the general adjoint); tables with one run only those.
template <typename T, bool POLYGON = false>
OLB_HD bool aperture_inside(const T* prog, int len, T x, T y) {
  uint32_t stack = 0;  // bit stack, top at bit 0
  int i = 0;
  while (i < len) {
    int op = (int)prog[i];
    bool v;
    if (op == OLB_AP_RADIAL) {
      T r2 = o_fma(x, x, y * y);
      v = (r2 <= prog[i + 1] * prog[i + 1]) && (r2 >= prog[i + 2] * prog[i + 2]);
      i += 3;
    } else if (op == OLB_AP_OFFSET_RADIAL) {
      T dx = x - prog[i + 3], dy = y - prog[i + 4];
      T r2 = o_fma(dx, dx, dy * dy);
      v = (r2 <= prog[i + 1] * prog[i + 1]) && (r2 >= prog[i + 2] * prog[i + 2]);
      i += 5;
    } else if (op == OLB_AP_RECT) {
      v = (prog[i + 1] <= x) && (x <= prog[i + 2]) && (prog[i + 3] <= y) && (y <= prog[i + 4]);
      i += 5;
    } else if (op == OLB_AP_ELLIPSE) {
      T dx = x - prog[i + 3], dy = y - prog[i + 4];
      T a = prog[i + 1], b = prog[i + 2];
      v = (o_div(dx * dx, a * a) + o_div(dy * dy, b * b)) <= (T)1;
      i += 5;
    } else if (POLYGON && op == OLB_AP_POLYGON) {
      v = polygon_inside(prog + i, x, y);
      i += PG_LEN;
    } else {
      bool b_ = stack & 1u, a_ = (stack >> 1) & 1u;
      stack >>= 2;
      v = op == OLB_AP_UNION ? (a_ || b_) : op == OLB_AP_INTERSECT ? (a_ && b_) : (a_ && !b_);
      i += 1;
    }
    stack = (stack << 1) | (v ? 1u : 0u);
  }
  return stack & 1u;
}


// ---- polarization (PolarizedRays.update, polarized_rays.py:136-202; JonesFresnel, jones.py:71-117) ----
template <typename T> struct Cx { T re, im; };
template <typename T> OLB_HD Cx<T> c_mul(Cx<T> a, Cx<T> b) { return {a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re}; }
template <typename T> OLB_HD Cx<T> c_div(Cx<T> a, Cx<T> b) {
  T d = o_rcp(o_fma(b.re, b.re, b.im * b.im));
  return {(a.re * b.re + a.im * b.im) * d, (a.im * b.re - a.re * b.im) * d};
}

template <typename T> OLB_HD Cx<T> c_add(Cx<T> a, Cx<T> b) { return {a.re + b.re, a.im + b.im}; }
template <typename T> OLB_HD Cx<T> c_sub(Cx<T> a, Cx<T> b) { return {a.re - b.re, a.im - b.im}; }
template <typename T> OLB_HD Cx<T> c_rcp(Cx<T> a) {
  T d = o_rcp(o_fma(a.re, a.re, a.im * a.im));
  return {a.re * d, -a.im * d};
}
// Principal square root, computed without cancellation.  A zero imaginary part takes the upper branch: the
// reference's X = nr^2 - k^2 - (n0 sin)^2 - 2i nr k never carries -0 there (0 - (+0) = +0 in numpy).
template <typename T> OLB_HD Cx<T> c_sqrt(Cx<T> z) {
  const T m = o_sqrt(o_fma(z.re, z.re, z.im * z.im));
  if (z.re >= 0) {
    const T t = o_sqrt((m + z.re) * (T)0.5);
    return {t, t == 0 ? (T)0 : o_div(z.im, 2 * t)};
  }
  const T t = o_sqrt((m - z.re) * (T)0.5);
  return {o_div(o_abs(z.im), 2 * t), z.im < 0 ? -t : t};
}
// sin(pi a), cos(pi a): the argument reduction of sincospi is exact and needs no reduction table in device memory
#if defined(__CUDA_ARCH__)
OLB_HD void o_sincospi(double a, double* s, double* c) { sincospi(a, s, c); }
OLB_HD void o_sincospi(float a, float* s, float* c) { sincospif(a, s, c); }
#else
template <typename T> inline void o_sincospi(T a, T* s, T* c) {
  const T r = a - 2 * std::rint(a / 2);   // exact: a - 2k, |r| <= 1
  *s = std::sin((T)M_PI * r);
  *c = std::cos((T)M_PI * r);
}
#endif

// Thin-film stack (OLB_COAT_THIN_FILM; thin_film/core.py:_tmm_coh): the Jones diagonal (js, jp) of one ray for both
// polarizations at once.  `hdr` is the prepared header (olb_prep.h, CO_*), `c2` = cos^2(aoi) (NaN for an unknown
// wavelength).  The incident medium's own X0 = n0~^2 cos^2 is formed from c2 directly: written as n0~^2 - n0~^2 sin^2
// it cancels near grazing incidence (in fp32 t_s was off by 2 % at 89.95 degrees).  Each characteristic matrix is carried scaled by e^{-|Im delta|} -- r is a ratio of degree-1 forms in
// (A, B, C, D) and does not see the scale, t is multiplied back by e^{-sum |Im delta|} -- so an absorbing layer with
// a large Im delta neither overflows cosh / sinh nor turns the products into inf / inf.
template <typename T>
OLB_HD void thin_film_jones(const T* hdr, int widx, T c2, bool reflect, Cx<T>& js, Cx<T>& jp) {
  const int L = (int)hdr[CO_L];
  const T* rec = hdr - (int)hdr[CO_BACK] + (int)hdr[CO_STRIDE] * widx;
  const T Y = (T)FILM_Y, iY = (T)(1.0 / FILM_Y);
  const T s2 = 1 - c2;
  const T n0r = rec[0] * s2, n0i = rec[1] * s2;   // (n0~ sin theta0)^2
  // X = A - (n0~ sin)^2 - iB, sqrt(X) = n~ cos theta;  eta_s = Y sqrt(X), eta_p = Y conj(n~)^2 / sqrt(X)
  // incident medium: X0 = A0 - iB0 - (A0 + iB0) sin^2 = A0 cos^2 - i B0 (1 + sin^2)
  const Cx<T> q0 = c_sqrt(Cx<T>{rec[0] * c2, (T)0 - rec[1] * (2 - c2)});
  const Cx<T> qs = c_sqrt(Cx<T>{rec[2] - n0r, (T)0 - n0i - rec[3]});
  const Cx<T> e0s = {Y * q0.re, Y * q0.im}, ess = {Y * qs.re, Y * qs.im};
  const Cx<T> e0p = c_mul(Cx<T>{Y * rec[0], -Y * rec[1]}, c_rcp(q0));
  const Cx<T> esp = c_mul(Cx<T>{Y * rec[2], -Y * rec[3]}, c_rcp(qs));
  Cx<T> As = {1, 0}, Bs = {0, 0}, Cs = {0, 0}, Ds = {1, 0};
  Cx<T> Ap = {1, 0}, Bp = {0, 0}, Cp = {0, 0}, Dp = {1, 0};
  T E = 0;
  for (int l = 0; l < L; ++l) {
    const T* ly = rec + CO_REC + CO_LAYER * l;
    const Cx<T> q = c_sqrt(Cx<T>{ly[1] - n0r, (T)0 - n0i - ly[2]});
    // delta = 2 pi d / lambda * sqrt(X) = pi (dr + i di)
    const T dr = ly[0] * q.re, di = (T)M_PI * (ly[0] * q.im);
    T sr, cr;
    o_sincospi(dr, &sr, &cr);
    const T adi = o_abs(di), e = o_exp(-2 * adi);
    const T ch = (1 + e) * (T)0.5, sh = (di < 0 ? (T)-0.5 : (T)0.5) * (1 - e);   // cosh, sinh times e^{-|di|}
    E += adi;
    const Cx<T> c = {cr * ch, -sr * sh};                // cos delta
    const Cx<T> is = {-cr * sh, sr * ch};               // i sin delta
    const Cx<T> iq = c_rcp(q);
    // s: i sin / eta = i sin / (Y q),  i eta sin = i sin Y q
    const Cx<T> mBs = c_mul(is, Cx<T>{iq.re * iY, iq.im * iY}), mCs = c_mul(is, Cx<T>{Y * q.re, Y * q.im});
    // p: i sin / eta_p = i sin q / (Y conj(n~)^2),  i eta_p sin = i sin Y conj(n~)^2 / q
    const Cx<T> mBp = c_mul(is, c_mul(q, Cx<T>{ly[3], ly[4]}));
    const Cx<T> mCp = c_mul(is, c_mul(Cx<T>{Y * ly[1], -Y * ly[2]}, iq));
    Cx<T> a = c_add(c_mul(As, c), c_mul(Bs, mCs)), b = c_add(c_mul(As, mBs), c_mul(Bs, c));
    Cx<T> cc = c_add(c_mul(Cs, c), c_mul(Ds, mCs)), d = c_add(c_mul(Cs, mBs), c_mul(Ds, c));
    As = a; Bs = b; Cs = cc; Ds = d;
    a = c_add(c_mul(Ap, c), c_mul(Bp, mCp)); b = c_add(c_mul(Ap, mBp), c_mul(Bp, c));
    cc = c_add(c_mul(Cp, c), c_mul(Dp, mCp)); d = c_add(c_mul(Cp, mBp), c_mul(Dp, c));
    Ap = a; Bp = b; Cp = cc; Dp = d;
  }
  const T sc = o_exp(-E);
  // denom = eta0 (A + etas B) + C + etas D ;  r = (eta0 (A + etas B) - C - etas D) / denom ;  t = conj(2 eta0 / denom)
  auto rt = [&](Cx<T> e0, Cx<T> es, Cx<T> A, Cx<T> B, Cx<T> C, Cx<T> D, Cx<T>& rr, Cx<T>& tt) {
    const Cx<T> u = c_mul(e0, c_add(A, c_mul(es, B))), v = c_add(C, c_mul(es, D));
    Cx<T> den = c_add(u, v);
    if (den.re == 0 && den.im == 0) den = {(T)1e-30, (T)0};
    const Cx<T> id = c_rcp(den);
    rr = c_mul(c_sub(u, v), id);
    const Cx<T> t2 = c_mul(Cx<T>{2 * e0.re, 2 * e0.im}, id);
    tt = {t2.re * sc, -t2.im * sc};
  };
  Cx<T> rs, ts, rp, tp;
  rt(e0s, ess, As, Bs, Cs, Ds, rs, ts);
  rt(e0p, esp, Ap, Bp, Cp, Dp, rp, tp);
  if (reflect) { js = rs; jp = {-rp.re, -rp.im}; }
  else { js = ts; jp = tp; }
}

// P := O_out * J * O_in * P for one ray.  k0 = (L0,M0,N0), k1 = (L,M,N) in the surface's local
// frame (the reference mixes local frames across tilted surfaces; reproduced).  `cosi` = |n.k0|.
// The matrix lives wherever the caller keeps it: element q (q = 2 (3 row + col) + {0: Re, 1: Im}) at P[q * ps] --
// the kernel holds it in shared memory ([q][thread], conflict-free, ps = block size) so that the 18 values are
// not carried in registers across the geometry step; the host check passes Ray::P with ps = 1.
// JONES (kernels of tables with a thin-film / polarizer / retarder coating) adds those coatings and the general 2x2
// Jones block; `pool` and `bad` (NaN for an unknown wavelength) are read by it only.
template <typename T, bool JONES = false>
OLB_HD void polar_update(Ray<T>& r, T* P, int ps, const PrepSurface<T>& S, T ncoat, T cosi, const T* pool = nullptr,
                         T bad = 0) {
  const T k0[3] = {r.L0, r.M0, r.N0}, k1[3] = {r.L, r.M, r.N};
  // s = k0 x k1, with the reference's fallback when k0 || k1 (polarized_rays.py:151-163).  At an
  // index-matched surface (the image surface: n1 == n2) k1 == k0 and s must come out exactly 0.
  T s[3];
  o_cross(k0, k1, s);
  T mag = o_sqrt(o_fma(s[0], s[0], o_fma(s[1], s[1], s[2] * s[2])));
  if (mag == 0) {
    T pf[3] = {(T)0, k0[2], -k0[1]};                       // k0 x (1,0,0)
    if (o_fma(pf[1], pf[1], pf[2] * pf[2]) == 0) { pf[0] = -k0[2]; pf[1] = 0; pf[2] = k0[0]; }  // k0 x (0,1,0)
    o_cross(pf, k0, s);                                    // p_fallback x k0
    mag = o_sqrt(o_fma(s[0], s[0], o_fma(s[1], s[1], s[2] * s[2])));
  }
  T inv = o_rcp(mag);
  s[0] *= inv; s[1] *= inv; s[2] *= inv;
  T p0[3], p1[3];
  o_cross(k0, s, p0);
  o_cross(k1, s, p1);
  // Jones diagonal (js, jp, jk)
  Cx<T> js = {(T)1, (T)0}, jp = {(T)1, (T)0};
  T jk = 1;
  if (S.coating == OLB_COAT_FRESNEL) {
    // aoi = arccos(clip(|n.k0|)) (coatings.py:72-93): cos(aoi) = c, sin^2(aoi) = 1 - c^2
    T c = cosi > (T)1 ? (T)1 : cosi;
    T n = ncoat, n2 = n * n;
    T rad = n2 - o_fma(-c, c, (T)1);
    Cx<T> root = rad >= 0 ? Cx<T>{o_sqrt(rad), (T)0} : Cx<T>{(T)0, o_sqrt(-rad)};   // principal sqrt
    if (!(rad == rad)) root = Cx<T>{rad, (T)0};
    Cx<T> cc = {c, (T)0}, n2c = {n2 * c, (T)0};
    if (S.flags & OLB_SF_REFLECT) {
      js = c_div(Cx<T>{cc.re - root.re, -root.im}, Cx<T>{cc.re + root.re, root.im});
      Cx<T> pp = c_div(Cx<T>{n2c.re - root.re, -root.im}, Cx<T>{n2c.re + root.re, root.im});
      jp = {-pp.re, -pp.im};
      jk = -1;
    } else {
      js = c_div(Cx<T>{2 * c, (T)0}, Cx<T>{cc.re + root.re, root.im});
      jp = c_div(Cx<T>{2 * n * c, (T)0}, Cx<T>{n2c.re + root.re, root.im});
    }
  }
  Cx<T> Mx[9];
  if constexpr (JONES) {
    // general Jones block (J00 J01; J10 J11), J22 = jk
    Cx<T> j01 = {(T)0, (T)0}, j10 = {(T)0, (T)0};
    const T* hdr = pool + S.media_off - CO_HDR;
    if (S.coating == OLB_COAT_THIN_FILM) {
      // aoi = arccos(clip(|n.k0|)): cos^2(aoi) = c^2
      const T c = cosi > (T)1 ? (T)1 : cosi;
      const bool refl = (S.flags & OLB_SF_REFLECT) != 0;
      thin_film_jones(hdr, r.widx < 0 ? 0 : r.widx, c * c + bad, refl, js, jp);
      jk = refl ? (T)-1 : (T)1;
    } else if (S.coating == OLB_COAT_POLARIZER || S.coating == OLB_COAT_RETARDER) {
      // (a.s, a.p0) and (a.s, a.p1), each normalised, a zero norm taken as 1 (jones.py: JonesLinearPolarizer /
      // JonesLinearRetarder); both act the same on reflection and transmission
      const T ax = hdr[CO_AX], ay = hdr[CO_AX + 1], az = hdr[CO_AX + 2];
      const T ts = o_fma(ax, s[0], o_fma(ay, s[1], az * s[2]));
      const T tpi = o_fma(ax, p0[0], o_fma(ay, p0[1], az * p0[2]));
      T ni = o_sqrt(o_fma(ts, ts, tpi * tpi));
      if (ni == 0) ni = 1;
      const T usi = o_div(ts, ni), upi = o_div(tpi, ni);
      if (S.coating == OLB_COAT_POLARIZER) {
        const T tpo = o_fma(ax, p1[0], o_fma(ay, p1[1], az * p1[2]));
        T no = o_sqrt(o_fma(ts, ts, tpo * tpo));
        if (no == 0) no = 1;
        const T uso = o_div(ts, no), upo = o_div(tpo, no);
        js = {uso * usi, (T)0}; j01 = {uso * upi, (T)0}; j10 = {upo * usi, (T)0}; jp = {upo * upi, (T)0};
      } else {
        // e^{-+id/2} us^2 + e^{+-id/2} up^2 = cos(d/2) (us^2 + up^2) -+ i sin(d/2) (us^2 - up^2)
        const T ch = hdr[CO_COS], sh = hdr[CO_SIN];
        const T u2 = usi * usi, v2 = upi * upi;
        js = {ch * (u2 + v2), -sh * (u2 - v2)};
        jp = {ch * (u2 + v2), sh * (u2 - v2)};
        j01 = {(T)0, -2 * sh * usi * upi};
        j10 = j01;
      }
      jk = 1;
    }
    // M[a][b] = s_a (J00 s_b + J01 p0_b) + p1_a (J10 s_b + J11 p0_b) + J22 k1_a k0_b
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      const Cx<T> u = {o_fma(js.re, s[b], j01.re * p0[b]), o_fma(js.im, s[b], j01.im * p0[b])};
      const Cx<T> v = {o_fma(j10.re, s[b], jp.re * p0[b]), o_fma(j10.im, s[b], jp.im * p0[b])};
#pragma unroll
      for (int a = 0; a < 3; ++a)
        Mx[3 * a + b] = {o_fma(s[a], u.re, o_fma(p1[a], v.re, k1[a] * k0[b] * jk)), o_fma(s[a], u.im, p1[a] * v.im)};
    }
  } else {
  // M[r][c] = s_r js s_c + p1_r jp p0_c + k1_r jk k0_c      (o_out @ J @ o_in)
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      T ss = s[a] * s[b], pp = p1[a] * p0[b], kk = k1[a] * k0[b] * jk;
      Mx[3 * a + b] = {o_fma(ss, js.re, o_fma(pp, jp.re, kk)), o_fma(ss, js.im, pp * jp.im)};
    }
  }
  // P := M P, column by column
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    Cx<T> col[3] = {{P[(2 * c) * ps], P[(2 * c + 1) * ps]}, {P[(2 * (3 + c)) * ps], P[(2 * (3 + c) + 1) * ps]},
                    {P[(2 * (6 + c)) * ps], P[(2 * (6 + c) + 1) * ps]}};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      Cx<T> v = c_mul(Mx[3 * a], col[0]);
      Cx<T> w1 = c_mul(Mx[3 * a + 1], col[1]);
      Cx<T> w2 = c_mul(Mx[3 * a + 2], col[2]);
      P[(2 * (3 * a + c)) * ps] = v.re + w1.re + w2.re;
      P[(2 * (3 * a + c) + 1) * ps] = v.im + w1.im + w2.im;
    }
  }
}

// PolarizedRays.update_intensity (optiland/rays/polarized_rays.py:122-133 with _get_3d_electric_field :204-233):
//   p = (k x xhat) / |k x xhat|,  s = p x k   (k = LAUNCH direction; the reference raises when k || xhat)
//   E0 = ax s + ay p  with the complex amplitudes ax = Ex e^{i phase_x}, ay = Ey e^{i phase_y}
//   i  = sum_states |P E0|^2 * i0 / n_states ;  unpolarized light = the two states (ax, ay) = (1, 0) and (0, 1).
// mode 1: one polarized state (ax, ay given as re / im pairs); mode 2: unpolarized.
template <typename T>
OLB_HD T polarized_intensity(const T* P, int ps, T kx, T ky, T kz, T i0, int mode, const T* ax, const T* ay, int& status) {
  // k x (1, 0, 0) = (0, kz, -ky)
  const T nrm = o_sqrt(o_fma(kz, kz, ky * ky));
  if (nrm == 0) status |= OLB_ST_K_PARALLEL_X;
  const T inv = o_rcp(nrm);
  const T pv[3] = {(T)0, kz * inv, -ky * inv};
  const T k[3] = {kx, ky, kz};
  T sv[3];
  o_cross(pv, k, sv);
  T total = 0;
  const int n_states = mode == 2 ? 2 : 1;
  for (int st = 0; st < n_states; ++st) {
    // amplitudes of this state
    const T axr = mode == 2 ? (st == 0 ? (T)1 : (T)0) : ax[0], axi = mode == 2 ? (T)0 : ax[1];
    const T ayr = mode == 2 ? (st == 0 ? (T)0 : (T)1) : ay[0], ayi = mode == 2 ? (T)0 : ay[1];
    T er[3], ei[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) { er[c] = o_fma(axr, sv[c], ayr * pv[c]); ei[c] = o_fma(axi, sv[c], ayi * pv[c]); }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      T re = 0, im = 0;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const T pr = P[(2 * (3 * a + c)) * ps], pi = P[(2 * (3 * a + c) + 1) * ps];
        re += pr * er[c] - pi * ei[c];
        im += pr * ei[c] + pi * er[c];
      }
      total += o_fma(re, re, im * im);
    }
  }
  return total * i0 / (T)n_states;
}

// Phase-profile interaction (PhaseInteractionModel.interact_real_rays, phase_interaction_model.py:45-124): the
// generalized Snell's law with the geometry's UNALIGNED normal n (include/olb.h, OLB_INTERACT_*).  The wave vectors
// are carried in units of k0 (k / k0, grad phi / k0), which leaves the direction unchanged and keeps every term O(1)
// in fp32.  `n1` is material_pre's index (NaN for an unknown wavelength).  Efficiency is applied by the caller after
// the coating step, as in the reference.
template <typename T>
OLB_HD void phase_interact(Ray<T>& r, const PrepSurface<T>& S, const T* pool, T nx, T ny, T nz, T n1) {
  const T* ph = pool + S.phase_off;
  const int nt = (int)ph[PH_NT];
  const T* c = ph + PH_P;
  const T* wl = c + (S.phase == OLB_INTERACT_PHASE_RADIAL ? 2 * nt : nt) + 2 * (r.widx < 0 ? 0 : r.widx);
  const T ik0 = wl[0], n2 = wl[1] + (n1 - n1);   // (n1 - n1: NaN for an unknown wavelength, 0 otherwise)
  T phi, gx, gy;
  if (S.phase == OLB_INTERACT_PHASE_RADIAL) {
    // phi = sum a_p r^(2p), grad phi = (x, y) sum 2p a_p r^(2p-2): Horner in r^2, no division (0 on axis)
    const T r2 = o_fma(r.x, r.x, r.y * r.y);
    T v = 0, d = 0;
    for (int p = nt - 1; p >= 0; --p) {
      v = o_fma(v, r2, c[p]);
      d = o_fma(d, r2, c[nt + p]);
    }
    phi = v * r2;
    gx = d * r.x;
    gy = d * r.y;
  } else if (S.phase == OLB_INTERACT_PHASE_LINEAR) {
    phi = o_fma(c[0], r.x, c[1] * r.y);
    gx = c[0];
    gy = c[1];
  } else {
    phi = c[0];
    gx = 0;
    gy = 0;
  }
  // G = grad phi - (grad phi . n) n ;  k_par = k_in - (k_in . n) n + G  (grad phi has no z component)
  gx *= ik0; gy *= ik0;
  const T gdn = o_fma(gx, nx, gy * ny);
  const T ax = n1 * r.L, ay = n1 * r.M, az = n1 * r.N;
  const T kdn = o_fma(ax, nx, o_fma(ay, ny, az * nz));
  const T px = o_fma(-kdn, nx, ax) + o_fma(-gdn, nx, gx);
  const T py = o_fma(-kdn, ny, ay) + o_fma(-gdn, ny, gy);
  const T pz = o_fma(-kdn, nz, az) - gdn * nz;
  T R2 = o_fma(n2, n2, -o_fma(px, px, o_fma(py, py, pz * pz)));
  if (R2 < 0) {           // evanescent: clipped, and a finite grazing direction (R^2 := 0; NaN stays NaN)
    r.i = 0;
    R2 = 0;
  }
  const T al = (S.flags & OLB_SF_REFLECT) ? -o_sqrt(R2) : o_sqrt(R2);
  const T kx = o_fma(al, nx, px), ky = o_fma(al, ny, py), kz = o_fma(al, nz, pz);
  const T inv = o_rsqrt(o_fma(kx, kx, o_fma(ky, ky, kz * kz)));
  r.L = kx * inv;
  r.M = ky * inv;
  r.N = kz * inv;
  accumulate_opd(r, -phi * ik0);   // opd += -phi / k0 (signed)
}

// The surface step.  FEAT gates code that most systems never need (register pressure, code
// size); KIND (0 plane, 1 sphere/conic closed form, 2 Newton family) is resolved by the caller
// ONCE per surface, outside the per-ray loop, so the hot loop carries no geometry branches.
enum { KIND_PLANE = 0, KIND_CONIC = 1, KIND_NEWTON = 2, KIND_ASPHERE = 3,   // NEWTON: any family (generic loop); ASPHERE: even / odd only (fused loop)
       KIND_GRID = 4 };                                                    // grid sag (FEAT_GRID kernels only)

// Ruled-grating interaction (DiffractiveInteractionModel.interact_real_rays, diffractive_model.py:28-61, with
// RealRays.gratingdiffract): the vector form of include/olb.h (OLB_INTERACT_GRATING), which is algebraically the
// reference's expanded expression divided through by the projected period, so every term is O(1) in fp32.  (nx, ny,
// nz) is the geometry's unaligned normal; `n1` is material_pre's index (NaN for an unknown wavelength).  KIND is
// KIND_PLANE (PlaneGrating) or KIND_CONIC (StandardGratingGeometry).  The reference's quirks stay: a reflective
// grating returns the negative of the physical direction, an evanescent order (Q < 0) leaves NaN direction cosines
// and the intensity unchanged, and no OPD term is added.
template <typename T, int KIND>
OLB_HD void grating_interact(Ray<T>& r, const PrepSurface<T>& S, const T* pool, T nx, T ny, T nz, T n1) {
  const T* gb = pool + S.phase_off + PH_P;
  const T* wl = gb + GR_WL + 2 * (r.widx < 0 ? 0 : r.widx);
  const T mld = wl[0], n2 = wl[1] + (n1 - n1);   // (n1 - n1: NaN for an unknown wavelength, 0 otherwise)
  // grating vector f, from the unaligned normal (plane_grating.py:113-132, standard_grating.py:102-256)
  T fx, fy, fz;
  if (KIND == KIND_PLANE) {
    fx = -gb[GR_SIN]; fy = gb[GR_COS]; fz = 0;
  } else {
    // groove tangent t = (1, tan a, dz/dx along the groove) with dz/dx = -(nx + tan a ny) / nz on the conic; scaled
    // by -nz > 0 (the conic normal points to -z), which f = -normalise(n x t) does not see
    const T ta = gb[GR_TAN];
    const T tx = -nz, ty = -nz * ta, tz = o_fma(ta, ny, nx);
    const T cx = o_fma(ny, tz, -nz * ty), cy = o_fma(nz, tx, -nx * tz), cz = o_fma(nx, ty, -ny * tx);
    const T inv = -o_rsqrt(o_fma(cx, cx, o_fma(cy, cy, cz * cz)));
    fx = cx * inv; fy = cy * inv; fz = cz * inv;
  }
  const T g = mld * o_sqrt(o_fma(fx, fx, fy * fy));   // m lambda / (d / sqrt(fx^2 + fy^2))
  // normal aligned with the incoming ray (real_rays.py:535-571; sign(0) = 0, sign(NaN) = NaN)
  const T dot = o_fma(r.L, nx, o_fma(r.M, ny, r.N * nz));
  const T sg = dot > 0 ? (T)1 : (dot < 0 ? (T)-1 : dot);
  const T mx = nx * sg, my = ny * sg, mz = nz * sg;
  const T ax = o_fma(g, fx, n1 * r.L), ay = o_fma(g, fy, n1 * r.M), az = o_fma(g, fz, n1 * r.N);
  const T nn = o_fma(mx, mx, o_fma(my, my, mz * mz));
  const T adn = o_fma(ax, mx, o_fma(ay, my, az * mz));
  // T = a |n|^2 - (a . n) n ;  Q = n2^2 |n|^2 - |a x n|^2
  const T tvx = o_fma(ax, nn, -adn * mx), tvy = o_fma(ay, nn, -adn * my), tvz = o_fma(az, nn, -adn * mz);
  const T qx = o_fma(ay, mz, -az * my), qy = o_fma(az, mx, -ax * mz), qz = o_fma(ax, my, -ay * mx);
  const T Q = o_fma(n2 * n2, nn, -o_fma(qx, qx, o_fma(qy, qy, qz * qz)));
  const T sq = gb[GR_SGN] * o_sqrt(Q);                  // NaN when evanescent (the reference's behaviour)
  const T sv = (S.flags & OLB_SF_REFLECT) ? (T)-1 : (T)1;
  const T kx = o_fma(sq, mx, sv * tvx), ky = o_fma(sq, my, sv * tvy), kz = o_fma(sq, mz, sv * tvz);
  const T inv = o_rsqrt(o_fma(kx, kx, o_fma(ky, ky, kz * kz)));
  r.L = kx * inv;
  r.M = ky * inv;
  r.N = kz * inv;
}

// BSDF scatter (include/olb.h OLB_SF_BSDF), defined in olb_bsdf.cuh: compiled only into FEAT_BSDF kernels.
template <typename T>
OLB_HD void bsdf_scatter(Ray<T>& r, const T* bs, T nx, T ny, T nz, int& status);

template <typename T, uint32_t FEAT, int KIND>
OLB_HD void surface_step_k(Ray<T>& r, const PrepSurface<T>& S, const T* pool, bool from_global, int& status,
                           T* Pm = nullptr, int Pstride = 1) {
  // -- localize (coordinate_system.py:73-89), from global or from the previous local frame
  if (FEAT & FEAT_ROT) {
    if (from_global) apply_affine(S.Ag, S.bg, (S.flags & PSF_ROT_IN_G) != 0, r.x, r.y, r.z, r.L, r.M, r.N);
    else apply_affine(S.Ar, S.br, (S.flags & PSF_ROT_IN_R) != 0, r.x, r.y, r.z, r.L, r.M, r.N);
  } else {
    const T* b = from_global ? S.bg : S.br;
    r.x += b[0]; r.y += b[1]; r.z += b[2];
  }
  const T* med = pool + S.media_off + MED_STRIDE * (r.widx < 0 ? 0 : r.widx);
  const T bad = r.widx < 0 ? (T)NAN : (T)0;  // unknown wavelength -> NaN in band

  // -- distance
  T t;
  T nfx = 0, nfy = 0;                                   // Newton family: slopes at the hit point
  if (KIND == KIND_PLANE) {
    t = -o_div(r.z, r.N);                               // plane.py:72-88
  } else if (KIND == KIND_CONIC) {
    t = conic_distance(r.x, r.y, r.z, r.L, r.M, r.N, S);
  } else if constexpr (KIND == KIND_GRID) {
    NewtonHit<T> h = grid_hit(r.x, r.y, r.z, r.L, r.M, r.N, S, pool);
    t = h.t; nfx = h.fx; nfy = h.fy;
  } else {
    NewtonHit<T> h = newton_hit<T, FEAT, KIND == KIND_ASPHERE>(r.x, r.y, r.z, r.L, r.M, r.N, &S, pool);
    t = h.t; nfx = h.fx; nfy = h.fy;
    status |= h.status;
  }
  // -- propagate (homogeneous.py:30-57) and OPD (standard_surface.py:244)
  r.x = o_fma(t, r.L, r.x);
  r.y = o_fma(t, r.M, r.y);
  r.z = o_fma(t, r.N, r.z);
  if (S.flags & OLB_SF_ABSORBING) r.i *= o_exp(-med[MED_ALPHA] * t);
  accumulate_opd(r, o_abs(t * (med[MED_N1] + bad)));

  // -- aperture clip (standard_surface.py:245-246; real_rays.py:154-161): NaN -> clipped
  if (S.flags & OLB_SF_APERTURE) {
    bool inside;
    if (S.flags & PSF_APER_RADIAL) {
      T r2 = o_fma(r.x, r.x, r.y * r.y);
      inside = (r2 <= pool[S.aper_off + 1]) && (r2 >= pool[S.aper_off + 2]);
    } else if (FEAT & FEAT_EXTRA) {
      inside = aperture_inside<T, (FEAT & FEAT_POLYGON) != 0>(pool + S.aper_off, S.aper_len, r.x, r.y);
    } else {
      inside = true;
    }
    if (!inside) r.i = 0;
  }

  // -- surface normal
  T nx, ny, nz;
  if (KIND == KIND_PLANE) {
    nx = 0; ny = 0; nz = 1;                             // plane.py:90-109
  } else if (KIND == KIND_CONIC) {
    // standard.py:150-175: (x, y, -denom)/ (denom * mag) with denom = R sqrt(1-(1+k) r2/R^2);
    // multiplied through by sqrt(.) >= 0 this is (x c, y c, -s) / sqrt(1 - k r2 c^2).
    T c = S.curv;
    T r2 = o_fma(r.x, r.x, r.y * r.y);
    T s = o_sqrt(o_fma(-S.kp1 * r2, c * c, (T)1));
    nx = r.x * c; ny = r.y * c; nz = -s;
    if (S.conic != 0) {
      T inv = o_rsqrt(o_fma(-S.conic * r2, c * c, (T)1));
      nx *= inv; ny *= inv; nz *= inv;
    }
  } else if constexpr (KIND == KIND_GRID) {
    // grid_sag.py:142-150: (-sx, -sy, 1) / |.|, the opposite sign to the other geometries (include/olb.h)
    T inv = o_rsqrt(o_fma(nfx, nfx, o_fma(nfy, nfy, (T)1)));
    nx = -nfx * inv; ny = -nfy * inv; nz = inv;
  } else {
    T inv = o_rsqrt(o_fma(nfx, nfx, o_fma(nfy, nfy, (T)1)));
    nx = nfx * inv; ny = nfy * inv; nz = -inv;
  }

  // -- interaction (refractive_reflective_model.py:32-55)
  if (FEAT & (FEAT_EXTRA | FEAT_POL)) { r.L0 = r.L; r.M0 = r.M; r.N0 = r.N; }
  bool phase = false;
  if constexpr ((FEAT & FEAT_PHASE) != 0) {
    // phase-profile surface (phase_interaction_model.py:45-132): replaces refract / reflect
    if (S.phase != OLB_INTERACT_REFRACT) {
      if constexpr ((FEAT & FEAT_GRATING) != 0 && (KIND == KIND_PLANE || KIND == KIND_CONIC)) {
        // ruled grating (diffractive_model.py:28-61): upload admits it on planes and conics only; its block has
        // efficiency 1, so the efficiency step below leaves i as the reference does
        if (S.phase == OLB_INTERACT_GRATING) grating_interact<T, KIND>(r, S, pool, nx, ny, nz, med[MED_N1] + bad);
        else phase_interact(r, S, pool, nx, ny, nz, med[MED_N1] + bad);
      } else {
        phase_interact(r, S, pool, nx, ny, nz, med[MED_N1] + bad);
      }
      phase = true;
    }
  }
  T dot = o_fma(r.L, nx, o_fma(r.M, ny, r.N * nz));
  if (phase) {
  } else if (S.flags & OLB_SF_REFLECT) {
    // real_rays.py:189-205 with the aligned normal: d - 2 |dot| sign(dot) n = d - 2 dot n
    T m2 = -2 * dot;
    r.L = o_fma(m2, nx, r.L);
    r.M = o_fma(m2, ny, r.M);
    r.N = o_fma(m2, nz, r.N);
  } else {
    // real_rays.py:163-187 + _align_surface_normal :535-571 (sign(0) = 0, sign(NaN) = NaN)
    T u = med[MED_U] + bad;
    T sgn = dot > 0 ? (T)1 : (dot < 0 ? (T)-1 : dot);
    T ad = o_abs(dot);
    T root = o_sqrt(o_fma(u * u, o_fma(ad, ad, (T)-1), (T)1));   // sqrt(1 - u^2 (1 - dot^2))
    T g = sgn * o_fma(-u, ad, root);
    // Index-matched surface (u == 1; every image surface): no deflection, exactly.  The
    // reference gets this from sqrt(x*x) == |x| in IEEE arithmetic; PolarizedRays.update needs
    // k1 == k0 bit-for-bit here (its s = k0 x k1 basis must fall back, polarized_rays.py:151-163).
    if (u == (T)1) g = (T)0 * dot;   // 0, or NaN when dot is NaN (NaN stays in band)
    r.L = o_fma(u, r.L, nx * g);
    r.M = o_fma(u, r.M, ny * g);
    r.N = o_fma(u, r.N, nz * g);
  }
  // -- scatter (interactions/base.py:115-116): about the outgoing direction, with the unaligned normal
  if constexpr ((FEAT & FEAT_BSDF) != 0) {
    if (S.flags & OLB_SF_BSDF) bsdf_scatter(r, pool + S.media_off - BS_LEN, nx, ny, nz, status);
  }
  // -- coating (interactions/base.py:111-128; coatings.py:164-237)
  if ((FEAT & FEAT_EXTRA) && S.coating == OLB_COAT_SIMPLE)
    r.i *= (S.flags & OLB_SF_REFLECT) ? S.coat_r : S.coat_t;
  // -- polarization: rays.update() / coating.interact -> rays.update(jones)  (base.py:119-128)
  // A SimpleCoating only scales the intensity: coating.interact never reaches rays.update(), so the P matrix
  // keeps its value across that surface (base.py:119-128: update() runs only in the no-coating branch).
  if (FEAT & FEAT_POL) {
    if (S.coating != OLB_COAT_SIMPLE)
      // (Pm is the caller's matrix storage -- never a pointer into `r`: taking r.P's address here would force the
      // whole ray state into local memory in the kernel)
      polar_update<T, (FEAT & FEAT_JONES) != 0>(r, Pm, Pstride, S, med[MED_CN] + bad,
                                                o_abs(o_fma(r.L0, nx, o_fma(r.M0, ny, r.N0 * nz))), pool, bad);
  }
  // -- phase profile efficiency (phase_interaction_model.py:129-130)
  if constexpr ((FEAT & FEAT_PHASE) != 0) {
    if (phase) r.i *= pool[S.phase_off + PH_EFF];
  }
}

// Runtime dispatch on the geometry kind (one ray).  The CUDA kernel does this dispatch once
// per surface around its per-ray loop instead; the host-check uses this form.
template <typename T, uint32_t FEAT>
OLB_HD void surface_step(Ray<T>& r, const PrepSurface<T>& S, const T* pool, bool from_global, int& status,
                         T* Pm = nullptr, int Pstride = 1) {
  if (S.kind == OLB_GEOM_PLANE) surface_step_k<T, FEAT, KIND_PLANE>(r, S, pool, from_global, status, Pm, Pstride);
  else if (S.kind == OLB_GEOM_STANDARD) surface_step_k<T, FEAT, KIND_CONIC>(r, S, pool, from_global, status, Pm, Pstride);
  else if constexpr ((FEAT & FEAT_GRID) != 0) {
    // grid-sag tables run the general kernel: the grid loop beside the one generic Newton loop
    if (S.kind == OLB_GEOM_GRID_SAG) surface_step_k<T, FEAT, KIND_GRID>(r, S, pool, from_global, status, Pm, Pstride);
    else surface_step_k<T, FEAT, KIND_NEWTON>(r, S, pool, from_global, status, Pm, Pstride);
  } else if constexpr ((FEAT & FEAT_NEWTON) != 0) {
    // without FEAT_FREEFORM every Newton surface of the table is an even / odd asphere: the fused loop; with
    // it, one generic loop serves all families (two loops in one kernel cost more I-cache than the fusion saves)
    if constexpr ((FEAT & FEAT_FREEFORM) != 0) surface_step_k<T, FEAT, KIND_NEWTON>(r, S, pool, from_global, status, Pm, Pstride);
    else surface_step_k<T, FEAT, KIND_ASPHERE>(r, S, pool, from_global, status, Pm, Pstride);
  }
}

// Local -> global for the record (coordinate_system.py:91-107).
template <typename T, uint32_t FEAT>
OLB_HD void to_global(const Ray<T>& r, const PrepSurface<T>& S, T& x, T& y, T& z, T& L, T& M, T& N) {
  if ((FEAT & FEAT_ROT) && (S.flags & OLB_SF_ROTATED)) {
    const T* R = S.R;
    x = o_fma(R[0], r.x, o_fma(R[1], r.y, o_fma(R[2], r.z, S.t[0])));
    y = o_fma(R[3], r.x, o_fma(R[4], r.y, o_fma(R[5], r.z, S.t[1])));
    z = o_fma(R[6], r.x, o_fma(R[7], r.y, o_fma(R[8], r.z, S.t[2])));
    L = o_fma(R[0], r.L, o_fma(R[1], r.M, R[2] * r.N));
    M = o_fma(R[3], r.L, o_fma(R[4], r.M, R[5] * r.N));
    N = o_fma(R[6], r.L, o_fma(R[7], r.M, R[8] * r.N));
  } else {
    x = r.x + S.t[0]; y = r.y + S.t[1]; z = r.z + S.t[2];
    L = r.L; M = r.M; N = r.N;
  }
}

}  // namespace olb


// =============================================================================================
// Reverse mode: adjoint of ONE surface step for ONE ray (the backward pass of config 3).
//
// The reference differentiates the eager graph of every element-wise op of section 3.1
// (optiland/optimization/optimizer/torch/base.py:96-156).  Here the adjoint is derived by hand:
//   * through the intersection by the implicit-function theorem on F(p0 + t d0; theta) = 0,
//     F = sag(x, y) - z  ->  dt = -(gradF.(dp0 + t dd0) + F_theta dtheta) / (gradF.d0)
//     (valid for the closed-form conic AND the Newton family: no unrolled iterations),
//   * through the normal via the Hessian of the rotationally symmetric sag,
//   * through Snell refraction / reflection, OPD, absorption and the pose translation.
// Supported: plane / sphere-conic / even asphere, any pose (tilt angles are constants of the adjoint),
// any aperture tree, simple coatings, one wavelength.  Everything is recomputed from the recorded rows (state
// after surface s-1 and position after surface s): the forward pass stores nothing extra.
// =============================================================================================
namespace olb {

enum { GP_TX = 0, GP_TY = 1, GP_TZ = 2, GP_CURV = 3, GP_CONIC = 4, GP_N1 = 5, GP_N2 = 6, GP_COEF = 7,
       GP_MAX_COEF = 12, GP_R = GP_COEF + GP_MAX_COEF, GP_COUNT = GP_R + 9,
       GP_SCALARS = GP_R };   // pg[] of surface_backward holds the first GP_SCALARS; the 9 dLoss/dR go to gR

template <typename T>
struct Adjoint { T x, y, z, L, M, N, i, opd; };

// What a polynomial-family surface (polynomial / Zernike: bivariate monomial tables S for the sag and D for the slopes)
// contributes to the gradient of its TABLES: dLoss/dS_ij = q xn^i yn^j and dLoss/dD_ij = ax i xn^(i-1) yn^j +
// ay j xn^i yn^(j-1).  The caller accumulates them (warp reduction in the kernel); the host maps the table gradients
// back to the user's coefficients, in which the tables are linear.
template <typename T> struct PolyAdj { T q, ax, ay, xn, yn; int active; };

// The geometry kinds whose sag / slope polynomials are bivariate monomial tables covered by the adjoint.  (A Chebyshev
// surface is expanded into monomials of (x / norm_x, y / norm_y) on upload, olb_prep.h: ONE table serves sag and slopes.)
OLB_HD bool poly_family_kind(int kind) {
  return kind == OLB_GEOM_POLYNOMIAL || kind == OLB_GEOM_ZERNIKE || kind == OLB_GEOM_CHEBYSHEV;
}

// Number of per-surface COEFFICIENT gradient slots behind the 7 scalars (pg[GP_COEF ..]): the even- / odd-asphere
// coefficients C_j, or the Clenshaw-basis coefficients b_m of a Forbes Q^bfs surface (the host maps dLoss/db to the user's
// a_m through the transposed change of basis, optiland_b200/autograd.py).
template <typename T>
OLB_HD int coef_grad_slots(const PrepSurface<T>& S) {
  return (S.kind == OLB_GEOM_EVEN_ASPHERE || S.kind == OLB_GEOM_ODD_ASPHERE || S.kind == OLB_GEOM_FORBES_QBFS) ? S.n_coef : 0;
}

// Forbes Clenshaw sum with its first TWO derivatives (adjoint only; forbes_q_sum serves the forward pass):
// alpha''_n = p alpha''_{n+1} - alpha''_{n+2} - 8 alpha'_{n+1}  (differentiate alpha'_n = p alpha'_{n+1} - alpha'_{n+2}
// - 4 alpha_{n+1} once more, dp/dx = -4), d2S/dx2 = 2 (alpha''_0 + alpha''_1).
template <typename T>
OLB_HD void forbes_q_sum2(const T* b, int nc, T x, T& S, T& dS, T& d2S) {
  const T p = (T)2 - (T)4 * x;
  T a0 = 0, a1 = 0, a2 = 0, d0 = 0, d1 = 0, d2 = 0, e0 = 0, e1 = 0, e2 = 0;
  for (int n = nc - 1; n >= 0; --n) {
    a0 = b[n] + p * a1 - a2;
    d0 = p * d1 - d2 - (T)4 * a1;
    e0 = p * e1 - e2 - (T)8 * d1;
    if (n > 0) { a2 = a1; a1 = a0; d2 = d1; d1 = d0; e2 = e1; e1 = e0; }
  }
  if (nc > 1) { S = (T)2 * (a0 + a1); dS = (T)2 * (d0 + d1); d2S = (T)2 * (e0 + e1); }
  else { S = (T)2 * a0; dS = (T)2 * d0; d2S = (T)2 * e0; }
}

// Table gradients of the polynomial families (olb_trace_bwd_* grad_tables): per surface two blocks (sag table S, slope table
// D) of GT_DIM x GT_DIM doubles, entry (i, j) <-> xn^i yn^j; tables wider than GT_DIM are outside the adjoint's scope.
enum { GT_DIM = 12, GT_BLOCK = GT_DIM * GT_DIM, GT_PER_SURFACE = 2 * GT_BLOCK };

// One ray's contribution to entry (i, j) of the two tables (see PolyAdj): xi = xn^i, xim = xn^(i-1), yj, yjm likewise.
template <typename T>
OLB_HD void poly_table_terms(const PolyAdj<T>& pa, int i, int j, T xi, T xim, T yj, T yjm, T& vS, T& vD) {
  vS = pa.q * xi * yj;
  vD = pa.ax * (T)i * xim * yj + pa.ay * (T)j * xi * yjm;
}

// pre: state BEFORE the surface in GLOBAL coordinates (record row s-1 or the launch state);
// (x1g, y1g, z1g): position AFTER the surface (record row s), global.
// a: in = dLoss/d(state after the surface, global); out = dLoss/d(state before it, global).
// pg[GP_SCALARS]: += dLoss/d(pose translation, curvature, conic, indices, asphere coefficients).
// gR (nullable; element q at gR[q * gR_stride], row-major 3x3): += dLoss/dR of a ROTATED pose -- R enters four
// times, p_loc = R^T (p - t), d_loc = R^T d, p' = R p_loc' + t, d' = R d_loc' -- from which the caller's
// autograd graph gets the gradients of the tilt angles.  It is written straight to the caller's accumulators
// (shared memory in the kernel) so that the 9 values never live in registers.
// Returns false (and leaves `a` zeroed) when the ray is not finite at this surface (NaN in band: no gradient).
// POLY == false compiles the polynomial-family branches out (tables without such surfaces: olb_trace_bwd_* keeps the
// register budget and speed it had before they existed).
template <typename T, bool POLY = true>
OLB_HD bool surface_backward(const PrepSurface<T>& S, const T* pool, T xg0, T yg0, T zg0, T L, T M, T N, T i0,
                             T x1g, T y1g, T z1g, Adjoint<T>& a, T* pg, T* gR = nullptr, int gR_stride = 1,
                             PolyAdj<T>* padj = nullptr) {
  // (L, M, N are taken by value: they are rotated into the local frame below for tilted poses)
  if (POLY && padj) padj->active = 0;
  const T* med = pool + S.media_off;  // one wavelength
  const T n1 = med[MED_N1], u = med[MED_U];
  const T n2 = o_div(n1, u);
  // local frame: p = R^T (pg - t), d = R^T dg  (rotation only for tilted poses; it is a constant of the
  // adjoint: gradients w.r.t. the tilt ANGLES are not produced, only those w.r.t. the translation t)
  const bool rot = (S.flags & OLB_SF_ROTATED) != 0;
  T x0 = xg0 - S.t[0], y0 = yg0 - S.t[1], z0 = zg0 - S.t[2];
  T x1 = x1g - S.t[0], y1 = y1g - S.t[1], z1 = z1g - S.t[2];
  const T dgx = L, dgy = M, dgz = N;                      // d in GLOBAL axes (for dLoss/dR)
  if (rot) {
    const T* R = S.R;
    T a0 = x0, b0 = y0, c0 = z0, a1 = x1, b1 = y1, c1 = z1, dl = L, dm = M, dn = N;
    x0 = R[0] * a0 + R[3] * b0 + R[6] * c0; y0 = R[1] * a0 + R[4] * b0 + R[7] * c0; z0 = R[2] * a0 + R[5] * b0 + R[8] * c0;
    x1 = R[0] * a1 + R[3] * b1 + R[6] * c1; y1 = R[1] * a1 + R[4] * b1 + R[7] * c1; z1 = R[2] * a1 + R[5] * b1 + R[8] * c1;
    L = R[0] * dl + R[3] * dm + R[6] * dn; M = R[1] * dl + R[4] * dm + R[7] * dn; N = R[2] * dl + R[5] * dm + R[8] * dn;
  }
  const T dd = o_fma(L, L, o_fma(M, M, N * N));
  const T t = o_div(o_fma(x1 - x0, L, o_fma(y1 - y0, M, (z1 - z0) * N)), dd);
  // t is built from every input (both intercepts and the direction): a NaN / inf in any of them makes it non-finite
  // (inf * 0 and inf - inf are NaN), so one test covers them all
  if (!(t - t == 0)) {
    a.x = a.y = a.z = a.L = a.M = a.N = a.i = a.opd = 0;
    return false;
  }
  // ---- recompute slopes, curvature terms -------------------------------------------------
  const bool plane = S.kind == OLB_GEOM_PLANE;
  const T r2 = o_fma(x1, x1, y1 * y1);
  T g = 0, gp = 0, sconic = 1, c = 0, kp1 = S.kp1;
  T asph_p = 0, asph_pp = 0;
  // Forbes Q^bfs departure P(w) = pre phi S (see below): the pieces shared by the slope factor and the parameter gradients
  T fb_a = 0, fb_pre = 0, fb_dpre = 0, fb_phi = 1, fb_dphi = 0, fb_da = 1, fb_S = 0, fb_dS = 0;
  bool fb_on = false;
  if (!plane) {
    c = S.curv;
    sconic = o_sqrt(o_fma(-kp1 * r2, c * c, (T)1));
    const T is = o_rcp(sconic);
    const T is3 = is * is * is;
    g = c * is;                                   // conic part of 2 S'(r2)
    gp = (T)0.5 * kp1 * c * c * c * is3;          // d/dr2
    if (S.kind == OLB_GEOM_EVEN_ASPHERE) {
      const T* cf = pool + S.coef_off;
      for (int j = S.n_coef - 1; j >= 0; --j) {   // Horner: sum 2(j+1) C_j r2^j and its r2-derivative
        asph_pp = o_fma(asph_pp, r2, asph_p);
        asph_p = o_fma(asph_p, r2, (T)(2 * (j + 1)) * cf[j]);
      }
      g += asph_p;
      gp += asph_pp;
    } else if (S.kind == OLB_GEOM_ODD_ASPHERE) {
      // sag = conic + sum C_i r^(i+1): slope factor g += sum (i+1) C_i r^(i-1),
      // d g / d r2 = sum (i+1)(i-1)/2 C_i r^(i-3)
      const T* cf = pool + S.coef_off;
      const T rr = o_sqrt(r2);
      if (rr > 0) {
        const T ir = o_rcp(rr);
        T pw = ir;                                 // r^(i-1)
        for (int j = 0; j < S.n_coef; ++j) {
          asph_p = o_fma((T)(j + 1) * cf[j], pw, asph_p);
          asph_pp = o_fma((T)0.5 * (T)((j + 1) * (j - 1)) * cf[j], pw * ir * ir, asph_pp);
          pw *= rr;
        }
      } else if (S.n_coef > 1) {
        // exactly on the vertex (the chief ray of an on-axis field): the slopes x g, y g vanish whatever g is, but the
        // Hessian g I + 2 g' x x^T of the sag does not -- its limit is the r^2 term's 2 C_1 (an r^1 term, C_0 != 0, is a
        // cone tip with no Hessian at all; an r^3 term's g' ~ 1/r multiplies x x^T = 0)
        asph_p = (T)2 * cf[1];
      }
      g += asph_p;
      gp += asph_pp;
    } else if (POLY && S.kind == OLB_GEOM_FORBES_QBFS) {
      // Forbes Q^bfs: sag = conic + P(w), P = pre(w) phi(w) S(a w) with w = r^2, a = 1 / norm_radius^2, pre = a w (1 - a w),
      // phi = sqrt(na / da), na = 1 - k c^2 w, da = 1 - (1 + k) c^2 w (forbes/geometry.py:187-366; forbes_sag above).
      // A rotationally symmetric sag: slope factor g = 2 sag'(w), so g += 2 P', gp += 2 P''  (the reference's analytic
      // slope IS the sag's derivative up to its 1e-12 guards, so the same g serves the normal and the
      // implicit-function theorem).  phi' = c^2 / (2 phi da^2); phi'' = c^4 / 4 (k (na da)^-3/2 + 3 (1 + k) na^-1/2 da^-5/2).
      // Outside the normalisation radius (and for an all-zero coefficient set) the surface is the bare conic, as in the
      // forward pass.  (POLY: Forbes tables run on the grad_tables variant of the kernel.)
      fb_a = S.inv_norm * S.inv_norm;
      const T usq = r2 * fb_a;
      if (S.n_coef > 0 && usq < (T)1) {
        fb_on = true;
        T d2S;
        forbes_q_sum2(pool + S.coef_off, S.n_coef, usq, fb_S, fb_dS, d2S);
        const T c2 = c * c;
        const T na = (T)1 - S.conic * c2 * r2;
        fb_da = (T)1 - kp1 * c2 * r2;
        fb_phi = o_sqrt(o_div(na, fb_da));
        const T ida = o_rcp(fb_da), ina = o_rcp(na);
        fb_dphi = o_div(c2 * ida * ida, (T)2 * fb_phi);
        const T rn = o_sqrt(ina), rd = o_sqrt(ida);             // na^-1/2, da^-1/2
        const T d2phi = (T)0.25 * c2 * c2 * (S.conic * rn * ina * rd * ida + (T)3 * kp1 * rn * rd * ida * ida);
        fb_pre = usq * ((T)1 - usq);
        fb_dpre = fb_a * ((T)1 - (T)2 * usq);
        const T d2pre = (T)-2 * fb_a * fb_a;
        const T Sp = fb_a * fb_dS, Spp = fb_a * fb_a * d2S;       // dS/dw, d2S/dw2
        g += (T)2 * (fb_dpre * fb_phi * fb_S + fb_pre * fb_dphi * fb_S + fb_pre * fb_phi * Sp);
        gp += (T)2 * (d2pre * fb_phi * fb_S + (T)2 * fb_dpre * fb_dphi * fb_S + (T)2 * fb_dpre * fb_phi * Sp
                      + fb_pre * d2phi * fb_S + (T)2 * fb_pre * fb_dphi * Sp + fb_pre * fb_phi * Spp);
      }
    }
  }
  T fx = x1 * g, fy = y1 * g;           // the reference's slope function (-> normal)
  T Fx = fx, Fy = fy;                   // the true gradient of the sag (-> implicit-function theorem)
  T jxx = 0, jxy = 0, jyx = 0, jyy = 0; // non-radial part of d(fx, fy)/d(x, y)
  T pax = 1, pay = 1, pxn = 0, pyn = 0;
  const bool polyfam = POLY && poly_family_kind(S.kind);
  if (polyfam) {
    const bool tri = (S.flags & PSF_POLY_TRI) != 0;
    pxn = x1 * S.inv_norm; pyn = y1 * S.inv_norm_y;
    T Ps, Sx, Sy;
    poly2_eval(pool + S.coef_off, S.poly_rows, S.poly_cols, tri, pxn, pyn, Ps, Sx, Sy);
    Fx = o_fma(Sx, S.inv_norm, fx);
    Fy = o_fma(Sy, S.inv_norm_y, fy);
    T Pd, Dx, Dy, Dxx, Dxy, Dyy;
    poly2_hess(pool + S.poly_d_off, S.poly_rows, S.poly_cols, tri, pxn, pyn, Pd, Dx, Dy, Dxx, Dxy, Dyy);
    T Dxs = Dx, Dys = Dy;
    if (S.kind == OLB_GEOM_ZERNIKE) {
      // the forward pass's regularised chain rule (newton_slopes); its factors a, b = 1 - O(1e-14 / rho) are treated
      // as constants of the adjoint
      const T eps = (T)1e-14;
      const T rho2 = o_fma(pxn, pxn, pyn * pyn);
      if (rho2 == 0) { Dxs = 0; Dys = 0; Dxx = 0; Dxy = 0; Dyy = 0; }
      else {
        const T rho = o_sqrt(rho2);
        const T a_ = o_div(rho, rho + eps), b_ = o_div(rho2, rho2 + eps), inv = o_rcp(rho2);
        const T xx = pxn * pxn, yy = pyn * pyn, xy = pxn * pyn * (a_ - b_);
        Dxs = o_fma(Dx, o_fma(a_, xx, b_ * yy), Dy * xy) * inv;
        Dys = o_fma(Dy, o_fma(a_, yy, b_ * xx), Dx * xy) * inv;
      }
    }
    // the reference's Chebyshev slope function leaves the chain-rule factors 1 / norm_x, 1 / norm_y out
    // (chebyshev.py:171-181; newton_slopes above reproduces it): the NORMAL is differentiated as the forward pass
    // computes it, the intersection (Fx, Fy) by the true gradient of the sag
    const bool cheb = S.kind == OLB_GEOM_CHEBYSHEV;
    pax = cheb ? (T)1 : S.inv_norm; pay = cheb ? (T)1 : S.inv_norm_y;
    fx = o_fma(Dxs, pax, fx);
    fy = o_fma(Dys, pay, fy);
    jxx = pax * S.inv_norm * Dxx; jxy = pax * S.inv_norm_y * Dxy;
    jyx = pay * S.inv_norm * Dxy; jyy = pay * S.inv_norm_y * Dyy;
  }
  // grid sag (POLY variant only): the bilinear cell's slopes serve the intersection and the normal; its Hessian is
  // sxx = syy = 0, sxy.  The forward normal (-sx, -sy, 1) / |.| is the negative of the (fx, fy, -1) / |.| used here,
  // which refraction and reflection (through the aligned normal) do not see.  The grid values are constants.
  const bool grid = POLY && S.kind == OLB_GEOM_GRID_SAG;
  if (grid) {
    T sxy;
    (void)grid_eval(S, pool, x1, y1, fx, fy, &sxy);
    Fx = fx; Fy = fy;
    jxy = sxy; jyx = sxy;
  }
  const T invG = plane ? (T)1 : o_rsqrt(o_fma(fx, fx, o_fma(fy, fy, (T)1)));
  // unit normal: plane (0,0,+1) (plane.py:90-109), otherwise (fx, fy, -1)/|.|
  const T nx = plane ? (T)0 : fx * invG, ny = plane ? (T)0 : fy * invG, nz = plane ? (T)1 : -invG;
  const T dot = o_fma(L, nx, o_fma(M, ny, N * nz));
  // total internal reflection: the forward pass's sqrt(1 - u^2 (1 - dot^2)) is NaN, so is the direction it records
  // (real_rays.py:163-187), while the intercept is finite.  The ray is NaN at this surface: no gradient -- the
  // partials below are NaN too, and even a zero adjoint times them would turn every accumulator NaN.  This drops the
  // gradient of the row's finite entries as well (intercept, intensity, OPD at this surface): the ray contributes
  // only through the rows in front of it.
  if (!(S.flags & OLB_SF_REFLECT) && u != (T)1 && !(o_fma(u * u, o_fma(dot, dot, (T)-1), (T)1) >= 0)) {
    a.x = a.y = a.z = a.L = a.M = a.N = a.i = a.opd = 0;
    return false;
  }

  // ---- adjoint of globalize ---------------------------------------------------------------
  pg[GP_TX] += a.x; pg[GP_TY] += a.y; pg[GP_TZ] += a.z;    // pg1 = R p1 + t
  T apx = a.x, apy = a.y, apz = a.z;            // d/d p1 (local)
  const bool wantR = rot && gR != nullptr;
  if (wantR) {
    // p' = R p1_loc + t and d' = R d_loc' :  dLoss/dR_ij += a(p')_i p1_loc_j + a(d')_i d_loc'_j, with the
    // outgoing local direction d_loc' recomputed from the interaction (a.* are still in global axes here)
    T ox, oy, oz;
    if (S.flags & OLB_SF_REFLECT) {
      ox = o_fma((T)-2 * dot, nx, L); oy = o_fma((T)-2 * dot, ny, M); oz = o_fma((T)-2 * dot, nz, N);
    } else {
      const T sgn = dot > 0 ? (T)1 : (dot < 0 ? (T)-1 : (T)0);
      const T aa = o_abs(dot);
      const T h = (u == (T)1) ? (T)0 : o_fma(-u, aa, o_sqrt(o_fma(u * u, o_fma(aa, aa, (T)-1), (T)1)));
      ox = o_fma(u, L, h * sgn * nx); oy = o_fma(u, M, h * sgn * ny); oz = o_fma(u, N, h * sgn * nz);
    }
    gR[0 * gR_stride] += o_fma(a.x, x1, a.L * ox); gR[1 * gR_stride] += o_fma(a.x, y1, a.L * oy); gR[2 * gR_stride] += o_fma(a.x, z1, a.L * oz);
    gR[3 * gR_stride] += o_fma(a.y, x1, a.M * ox); gR[4 * gR_stride] += o_fma(a.y, y1, a.M * oy); gR[5 * gR_stride] += o_fma(a.y, z1, a.M * oz);
    gR[6 * gR_stride] += o_fma(a.z, x1, a.N * ox); gR[7 * gR_stride] += o_fma(a.z, y1, a.N * oy); gR[8 * gR_stride] += o_fma(a.z, z1, a.N * oz);
  }
  if (rot) {
    const T* R = S.R;
    apx = R[0] * a.x + R[3] * a.y + R[6] * a.z; apy = R[1] * a.x + R[4] * a.y + R[7] * a.z; apz = R[2] * a.x + R[5] * a.y + R[8] * a.z;
    T gl = a.L, gm = a.M, gn = a.N;
    a.L = R[0] * gl + R[3] * gm + R[6] * gn; a.M = R[1] * gl + R[4] * gm + R[7] * gn; a.N = R[2] * gl + R[5] * gm + R[8] * gn;
  }
  T ai = a.i;
  if (S.coating == OLB_COAT_SIMPLE) ai *= (S.flags & OLB_SF_REFLECT) ? S.coat_r : S.coat_t;
  // ---- adjoint of the interaction ------------------------------------------------------------
  T adL, adM, adN, anx, any_, anz;
  if (S.flags & OLB_SF_REFLECT) {
    const T dn = o_fma(a.L, nx, o_fma(a.M, ny, a.N * nz));
    adL = o_fma((T)-2 * dn, nx, a.L); adM = o_fma((T)-2 * dn, ny, a.M); adN = o_fma((T)-2 * dn, nz, a.N);
    anx = (T)-2 * o_fma(dot, a.L, dn * L); any_ = (T)-2 * o_fma(dot, a.M, dn * M); anz = (T)-2 * o_fma(dot, a.N, dn * N);
  } else {
    const T sgn = dot > 0 ? (T)1 : (dot < 0 ? (T)-1 : (T)0);
    const T aa = o_abs(dot);
    const T mx = sgn * nx, my = sgn * ny, mz = sgn * nz;
    const T root = o_sqrt(o_fma(u * u, o_fma(aa, aa, (T)-1), (T)1));
    const T h = o_fma(-u, aa, root);
    const T ah = o_fma(a.L, mx, o_fma(a.M, my, a.N * mz));
    const T ir = o_rcp(root);
    T au = o_fma(a.L, L, o_fma(a.M, M, a.N * N)) - aa * ah + ah * u * o_fma(aa, aa, (T)-1) * ir;
    T adot = -u * ah + ah * u * u * aa * ir;
    if (u == (T)1) { au = o_fma(a.L, L, o_fma(a.M, M, a.N * N)) - aa * ah + ah * o_fma(aa, aa, (T)-1) * o_rcp(aa); adot = 0; }
    adL = o_fma(u, a.L, adot * mx); adM = o_fma(u, a.M, adot * my); adN = o_fma(u, a.N, adot * mz);
    const T amx = o_fma(h, a.L, adot * L), amy = o_fma(h, a.M, adot * M), amz = o_fma(h, a.N, adot * N);
    anx = sgn * amx; any_ = sgn * amy; anz = sgn * amz;
    pg[GP_N1] += o_div(au, n2);
    pg[GP_N2] -= o_div(au * u, n2);
  }
  // ---- adjoint of the normal (Hessian of the sag) -------------------------------------------
  T ax1 = 0, ay1 = 0, ag = 0;
  if (!plane) {
    const T an_n = o_fma(anx, nx, o_fma(any_, ny, anz * nz));
    const T afx = (anx - an_n * nx) * invG, afy = (any_ - an_n * ny) * invG;
    ag = o_fma(afx, x1, afy * y1);
    const T ar2 = ag * gp;
    ax1 = o_fma(afx, g, (T)2 * x1 * ar2);
    ay1 = o_fma(afy, g, (T)2 * y1 * ar2);
    if (polyfam || grid) {
      ax1 += o_fma(afx, jxx, afy * jyx);
      ay1 += o_fma(afx, jxy, afy * jyy);
      if (polyfam && padj) { padj->ax = afx * pax; padj->ay = afy * pay; }
    }
  }
  // ---- clip / absorption / OPD ------------------------------------------------------------------
  T at = 0;
  {
    bool inside = true;
    if (S.flags & OLB_SF_APERTURE)
      inside = (S.flags & PSF_APER_RADIAL) ? ((r2 <= pool[S.aper_off + 1]) && (r2 >= pool[S.aper_off + 2]))
                                           : aperture_inside<T, POLY>(pool + S.aper_off, S.aper_len, x1, y1);
    T E = 1;
    if (S.flags & OLB_SF_ABSORBING) { E = o_exp(-med[MED_ALPHA] * t); at -= ai * i0 * med[MED_ALPHA] * E * (inside ? (T)1 : (T)0); }
    ai = inside ? ai * E : (T)0;
    const T tn = t * n1;
    const T sg = tn > 0 ? (T)1 : (tn < 0 ? (T)-1 : (T)0);
    at = o_fma(a.opd * sg, n1, at);
    pg[GP_N1] += a.opd * sg * t;
  }
  // ---- propagate p1 = p0 + t d0 ---------------------------------------------------------------------
  apx += ax1; apy += ay1;
  adL = o_fma(t, apx, adL); adM = o_fma(t, apy, adM); adN = o_fma(t, apz, adN);
  at += o_fma(apx, L, o_fma(apy, M, apz * N));
  // ---- intersection (implicit function theorem) -------------------------------------------------------
  const T D = o_fma(Fx, L, o_fma(Fy, M, -N));
  const T q = -o_div(at, D);
  apx = o_fma(q, Fx, apx); apy = o_fma(q, Fy, apy); apz -= q;
  const T qt = q * t;
  adL = o_fma(qt, Fx, adL); adM = o_fma(qt, Fy, adM); adN -= qt;
  if (polyfam && padj) { padj->q = q; padj->xn = pxn; padj->yn = pyn; padj->active = 1; }
  if (!plane && !grid) {
    const T is = o_rcp(sconic), is3 = is * is * is, ops = (T)1 + sconic;
    // d sag / d c = r2 / (s (1+s)) ; d sag / d k = c^3 r2^2 / (2 s (1+s)^2)
    // d g / d c = 1 / s^3          ; d g / d k   = c^3 r2 / (2 s^3)
    const T c3 = c * c * c;
    pg[GP_CURV] += q * r2 * is * o_rcp(ops) + ag * is3;
    pg[GP_CONIC] += q * (T)0.5 * c3 * r2 * r2 * is * o_rcp(ops * ops) + ag * (T)0.5 * c3 * r2 * is3;
    if (S.kind == OLB_GEOM_EVEN_ASPHERE) {
      T pw = 1;                                  // r2^j
#pragma unroll
      for (int j = 0; j < GP_MAX_COEF; ++j) {    // compile-time bound: pg[] stays in registers
        if (j < S.n_coef) pg[GP_COEF + j] += q * pw * r2 + ag * (T)(2 * (j + 1)) * pw;  // d sag/dC_j = r2^(j+1); d g/dC_j = 2(j+1) r2^j
        pw *= r2;
      }
    } else if (S.kind == OLB_GEOM_ODD_ASPHERE) {
      const T rr = o_sqrt(r2);
      T pw = rr > 0 ? o_rcp(rr) : (T)0;          // r^(j-1); the slope term vanishes at r == 0 like the forward pass
      T pws = rr;                                // r^(j+1)
#pragma unroll
      for (int j = 0; j < GP_MAX_COEF; ++j) {
        if (j < S.n_coef) pg[GP_COEF + j] += q * pws + ag * (T)(j + 1) * pw;   // d sag/dC_j = r^(j+1); d g/dC_j = (j+1) r^(j-1)
        pw *= rr; pws *= rr;
      }
    } else if (POLY && fb_on) {
      // Forbes departure: curvature and conic enter P through phi only,
      //   dphi/dc = c w / (phi da^2),                      dphi/dk = c^4 w^2 / (2 phi da^2),
      //   dphi'/dc = c/(phi da^2) - c^3 w/(2 phi^3 da^4) + 2 (1+k) c^3 w/(phi da^3),
      //   dphi'/dk = -c^6 w^2/(4 phi^3 da^4) + c^4 w/(phi da^3),
      // dP/dtheta = pre S dphi/dtheta,  dP'/dtheta = (pre' S + pre S') dphi/dtheta + pre S dphi'/dtheta;  g carries 2 P'.
      const T w = r2, ida = o_rcp(fb_da), ida2 = ida * ida, iphi = o_rcp(fb_phi), iphi3 = iphi * iphi * iphi;
      const T c2 = c * c, c3 = c2 * c, c4 = c2 * c2;
      const T dphi_dc = c * w * ida2 * iphi;
      const T dphi_dk = (T)0.5 * c4 * w * w * ida2 * iphi;
      const T ddphi_dc = c * ida2 * iphi - (T)0.5 * c3 * w * ida2 * ida2 * iphi3 + (T)2 * kp1 * c3 * w * ida2 * ida * iphi;
      const T ddphi_dk = (T)-0.25 * c4 * c2 * w * w * ida2 * ida2 * iphi3 + c4 * w * ida2 * ida * iphi;
      const T Sp = fb_a * fb_dS;
      const T A = fb_dpre * fb_S + fb_pre * Sp, B = fb_pre * fb_S;
      pg[GP_CURV] += q * B * dphi_dc + ag * (T)2 * (A * dphi_dc + B * ddphi_dc);
      pg[GP_CONIC] += q * B * dphi_dk + ag * (T)2 * (A * dphi_dk + B * ddphi_dk);
      // the Clenshaw-basis coefficients: S = sum_m b_m B_m(usq), B_m = 2 (U_m + U_{m-1})(p), p = 2 - 4 usq,
      // U_0 = 1, U_1 = p, U_{m+1} = p U_m - U_{m-1}:  dP/db_m = pre phi B_m,  dP'/db_m = (pre' phi + pre phi') B_m + pre phi a B_m'
      const T p = (T)2 - (T)4 * w * fb_a;
      const T k0 = fb_pre * fb_phi, k1 = fb_dpre * fb_phi + fb_pre * fb_dphi;
      T Um1 = 0, U = 1, dUm1 = 0, dU = 0;        // U_{m-1}, U_m and their derivatives with respect to p
#pragma unroll
      for (int m = 0; m < GP_MAX_COEF; ++m) {
        if (m < S.n_coef) {
          const T Bm = (T)2 * (U + Um1), dBm = (T)-8 * (dU + dUm1);          // B_m and dB_m / d usq
          pg[GP_COEF + m] += q * k0 * Bm + ag * (T)2 * (k1 * Bm + k0 * fb_a * dBm);
        }
        const T Un = p * U - Um1, dUn = U + p * dU - dUm1;
        Um1 = U; U = Un; dUm1 = dU; dU = dUn;
      }
    }
  }
  // ---- localize p0 = pg0 - t -------------------------------------------------------------------------
  if (wantR) {   // p_loc = R^T (p - t), d_loc = R^T d :  dLoss/dR_ij += (p - t)_i a(p_loc)_j + d_i a(d_loc)_j
    const T q0x = xg0 - S.t[0], q0y = yg0 - S.t[1], q0z = zg0 - S.t[2];
    gR[0 * gR_stride] += o_fma(q0x, apx, dgx * adL); gR[1 * gR_stride] += o_fma(q0x, apy, dgx * adM); gR[2 * gR_stride] += o_fma(q0x, apz, dgx * adN);
    gR[3 * gR_stride] += o_fma(q0y, apx, dgy * adL); gR[4 * gR_stride] += o_fma(q0y, apy, dgy * adM); gR[5 * gR_stride] += o_fma(q0y, apz, dgy * adN);
    gR[6 * gR_stride] += o_fma(q0z, apx, dgz * adL); gR[7 * gR_stride] += o_fma(q0z, apy, dgz * adM); gR[8 * gR_stride] += o_fma(q0z, apz, dgz * adN);
  }
  if (rot) {   // back to global: ag = R a_local
    const T* R = S.R;
    T u0 = apx, u1 = apy, u2 = apz, v0 = adL, v1 = adM, v2 = adN;
    apx = R[0] * u0 + R[1] * u1 + R[2] * u2; apy = R[3] * u0 + R[4] * u1 + R[5] * u2; apz = R[6] * u0 + R[7] * u1 + R[8] * u2;
    adL = R[0] * v0 + R[1] * v1 + R[2] * v2; adM = R[3] * v0 + R[4] * v1 + R[5] * v2; adN = R[6] * v0 + R[7] * v1 + R[8] * v2;
  }
  pg[GP_TX] -= apx; pg[GP_TY] -= apy; pg[GP_TZ] -= apz;
  a.x = apx; a.y = apy; a.z = apz; a.L = adL; a.M = adM; a.N = adN; a.i = ai;  // a.opd passes through
  return true;
}

}  // namespace olb
#endif  // OLB_MATH_CUH_
