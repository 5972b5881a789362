// olb_prep.h -- device-side ("prepared") surface table and its host-side construction.
//
// The host table of include/olb.h (fp64, reference vocabulary) is turned once per
// upload into one contiguous blob per element type T (float / double):
//
//     [ PrepHeader ][ PrepSurface<T> x n_surf ][ T pool[...] ]
//
// which the trace kernel pulls into shared memory with a single TMA bulk copy.
// Everything that is uniform over rays is precomputed here in fp64: flattened poses
// and surface-to-surface relative transforms, curvature, index ratios n1/n2 per
// wavelength, Beer-Lambert coefficients, and the monomial form of Zernike sums.
//
// Reference data contract: SURVEY.md Appendix B; citations inline.
#ifndef OLB_PREP_H_
#define OLB_PREP_H_

#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/olb.h"

namespace olb {

// Feature bits: which code paths a table needs (selects the kernel instantiation).
enum : uint32_t {
  FEAT_ROT = 1u << 0,      // some surface has a rotated pose
  FEAT_NEWTON = 1u << 1,   // a Newton-iteration surface (alone: even / odd aspheres only)
  FEAT_EXTRA = 1u << 2,    // non-radial aperture programs, simple coatings, L0/M0/N0 output
  FEAT_POL = 1u << 3,      // polarized rays (P matrix) / Fresnel coatings
  FEAT_FREEFORM = 1u << 4, // polynomial / Zernike / Chebyshev / biconic / toroidal / Forbes surfaces (with NEWTON)
  FEAT_PHASE = 1u << 5,    // a phase-profile surface (PhaseInteractionModel): runs the general kernel + this
  FEAT_GRATING = 1u << 6,  // a ruled grating (DiffractiveInteractionModel): runs the general kernel + PHASE + this
  FEAT_JONES = 1u << 7,    // a thin-film / polarizer / retarder coating (with POL): the general polarized kernel +
                           // PHASE + GRATING + this
  FEAT_GRID = 1u << 8,     // a grid-sag surface: the general kernel (polarized: + JONES) + PHASE + GRATING + this
  FEAT_POLYGON = 1u << 9,  // a polygon in an aperture program: the grid-sag superset + this
  FEAT_BSDF = 1u << 10,    // a BSDF scatter (OLB_SF_BSDF): the polygon superset + this (unpolarized only)
  FEAT_Q2D = 1u << 11,     // a Forbes Q-2D surface: the general kernel (plain or polarized) + this, nothing else
};

// Prepared Forbes Q-2D block (PrepSurface::coef_off; n_coef = M, poly_rows = n0), elements of T:
//   {vertex slope x, vertex slope y, norm_radius, 0}, the m = 0 list in the Q-bfs Clenshaw basis (n0), then per m = 1 .. M
//   {na, nb, N = max(na, nb), 0}, N rows {A(n, m), B(n, m), C(n + 1, m)} of abc_q2d_clenshaw (qpoly.py:373-400), the
//   cosine list in the Clenshaw basis (na), the sine list (nb).  The blocks follow each other without padding.
enum { Q2_VX = 0, Q2_VY = 1, Q2_NORM = 2, Q2_HDR = 4, Q2_NA = 0, Q2_NB = 1, Q2_N = 2, Q2_MHDR = 4 };


// Prepared BSDF block of a surface with OLB_SF_BSDF: BS_LEN elements of T right BEFORE its prepared media block (the
// kernel finds it from PrepSurface::media_off alone; a BSDF table never runs the polarized kernels, whose coating
// header sits there instead): {kind, sigma, key bits 0-15, 16-31, 32-47, 48-63, 0, 0}.  The 64-bit Philox key is kept
// in 16-bit pieces, each exact in fp32, so both precisions draw with the same key.
enum { BS_KIND = 0, BS_SIGMA = 1, BS_KEY = 2, BS_LEN = 8 };

// Prepared block of a thin-film / polarizer / retarder coating: it sits right BEFORE the surface's prepared media
// block, so the kernel finds it from PrepSurface::media_off alone.  Its CO_HDR-element header ends at media_off:
//   thin film : {L, record stride, n_wl * stride, ...}; the records of wavelengths 0 .. n_wl-1 precede the header
//               (record j at header - n_wl * stride + j * stride): {A0, B0, As, Bs} of the incident medium and the
//               substrate, then per layer {2 d / lambda, A, B, Re, Im of 1 / (Y conj(n~)^2)}, where for n~ = n + ik
//               A = n^2 - k^2 and B = 2 n k (so n~^2 = A + iB and conj(n~)^2 = A - iB)
//   polarizer : {ax, ay, az}
//   retarder  : {ax, ay, az, cos(d/2), sin(d/2)}
enum { CO_HDR = 8, CO_L = 0, CO_STRIDE = 1, CO_BACK = 2, CO_AX = 0, CO_COS = 3, CO_SIN = 4, CO_REC = 4, CO_LAYER = 5 };
// thin-film admittance of free space, sqrt(eps0 / mu0) in siemens (thin_film/core.py:_admittance)
constexpr double FILM_Y = 0.002654418729832701370374020517935;

// Prepared phase block per surface (PrepSurface::phase_off), elements of T:
//   [PH_EFF] efficiency, [PH_NT] number of profile terms n, then from PH_P the profile terms:
//   constant {phi}; linear {Kx, Ky}; radial {a_1 .. a_n, 2 a_1, 4 a_2 .. 2n a_n} (value and gradient Horner
//   coefficients in r^2); then, per wavelength j, {1 / k0 = lambda_j * 1e-3 / (2 pi) (mm / rad), n2 of the
//   interaction (n1 when reflective, phase_interaction_model.py:53-56)}.
enum { PH_EFF = 0, PH_NT = 1, PH_P = 2 };
// Prepared grating block (OLB_INTERACT_GRATING), from PH_P: {sin alpha, cos alpha, tan alpha, sign(d)}, then per
// wavelength j {m lambda_j / d, n2 = material_post's index} (GR_WL + 2 j).
enum { GR_SIN = 0, GR_COS = 1, GR_TAN = 2, GR_SGN = 3, GR_WL = 4 };

// Prepared OLB_AP_POLYGON instruction, PG_LEN elements of T in the aperture program:
//   {opcode, [PG_NB] number of y-buckets, [PG_YMIN] min vy, [PG_YMAX] max vy, [PG_SCALE] buckets per unit y,
//    [PG_OFF] offset of the edge block from the opcode}
// A point with py < min vy or py >= max vy (or NaN) has `cond` false on every edge: outside, no edge is read.  The edge
// block, 16-byte aligned, is start[nb + 1] (padded to 4) and then the edge records {vx, vy, vy_next, slope}, grouped by
// bucket: bucket b holds records start[b] .. start[b + 1] - 1, every edge whose y-span reaches it (an edge that spans
// several buckets is repeated in each; horizontal edges, which never cross, are left out).  The bucket of a point is
// polygon_bucket() below, the SAME function that placed the edges; it is monotone in py, so an edge with
// lo <= py < hi lies in [bucket(lo), bucket(hi)] -- the scan of one bucket counts exactly the crossings the scan of all
// edges would.  Outlines of up to PG_LINEAR_MAX vertices get one bucket (a plain scan, every lane of a warp reading
// the same record); longer ones one bucket per PG_PER_BUCKET vertices, halved until the records are at most twice
// the edges (an outline of long zigzags would otherwise repeat every edge in every bucket).
enum { PG_NB = 1, PG_YMIN = 2, PG_YMAX = 3, PG_SCALE = 4, PG_OFF = 5, PG_LEN = 6, PG_REC = 4,
       PG_LINEAR_MAX = 16, PG_PER_BUCKET = 4 };

#if defined(__CUDACC__)
#define OLB_PREP_HD __host__ __device__ __forceinline__
#else
#define OLB_PREP_HD inline
#endif
template <typename T>
OLB_PREP_HD int polygon_bucket(T y, T ymin, T scale, int nb) {
  const int b = (int)((y - ymin) * scale);   // ymin <= y <= ymax: between 0 and nb (1 + rounding)
  return b < nb - 1 ? b : nb - 1;
}

struct PrepHeader {
  int32_t n_surf;
  int32_t n_wl;
  int32_t pool_len;     // in elements of T
  uint32_t features;    // FEAT_* needed by this table
  int32_t blob_bytes;   // total bytes of this blob (multiple of 16)
  int32_t elem_size;    // sizeof(T)
  int32_t pad[2];
};  // 32 bytes

// Media block per surface in the pool: n_wl records of MEDIA_STRIDE values each.
enum { MED_N1 = 0, MED_U = 1, MED_ALPHA = 2, MED_CN = 3, MED_STRIDE = 4 };
//   MED_N1    n1                           (OPD: standard_surface.py:244)
//   MED_U     n1 / n2                      (refract: real_rays.py:174)
//   MED_ALPHA 4*pi*k1/lambda * 1e3         (homogeneous.py:45-53)
//   MED_CN    coating n2 / coating n1      (jones.py:95)

template <typename T>
struct PrepSurface {
  int32_t kind;
  uint32_t flags;      // OLB_SF_* plus the PSF_* bits below
  int32_t n_coef;      // even/odd: number of coefficients
  int32_t coef_off;    // pool offset (elements of T)
  int32_t aper_off;
  int32_t aper_len;
  int32_t max_iter;
  int32_t coating;
  int32_t media_off;
  int32_t poly_rows;   // bivariate tables: rows (x powers) and cols (y powers)
  int32_t poly_cols;
  int32_t poly_d_off;  // pool offset of the derivative-source table (Zernike quirk)
  int32_t gslot;       // backward: first per-thread gradient accumulator slot of this surface
  int32_t gslots;      //           number of slots (7 + n_coef [+ 9 for a tilted pose]; 0 for NOOP)
  int32_t phase;       // OLB_INTERACT_* (0: refractive / reflective); read by FEAT_PHASE kernels only
  int32_t phase_off;   // pool offset of the prepared phase block (PH_* below)
  // (sizeof stays a multiple of 16 (256 / 448 bytes): the pool behind the array stays 16-byte aligned)
  // incoming transform from GLOBAL coordinates: p_loc = Ag * p + bg
  T Ag[9], bg[3];
  // incoming transform from the PREVIOUS surface's local frame: p_loc = Ar * p + br
  T Ar[9], br[3];
  // outgoing transform to global: p_glob = R * p_loc + t
  T R[9], t[3];
  T radius, curv, conic, kp1;   // curv = 1/radius (0 for infinite radius), kp1 = 1 + k
  T tol, coat_t, coat_r, inv_norm;  // inv_norm = 1 / norm_radius (Chebyshev: 1 / norm_x)
  T inv_norm_y, curv_y, kp1_y, r_rot;  // Chebyshev 1/norm_y; biconic cy, 1+ky; toroidal: c_yz, 1+k_yz, R_rot
};
// the pool starts right behind the PrepSurface array: 16-byte alignment of its (4-element aligned) blocks needs this
static_assert(sizeof(PrepSurface<float>) % 16 == 0 && sizeof(PrepSurface<double>) % 16 == 0, "PrepSurface must keep the pool 16-byte aligned");
static_assert(sizeof(PrepHeader) % 16 == 0, "PrepHeader must keep the table 16-byte aligned");


enum : uint32_t {
  PSF_ROT_IN_G = 1u << 8,    // Ag != I
  PSF_ROT_IN_R = 1u << 9,    // Ar != I
  PSF_RADIUS_INF = 1u << 10, // StandardGeometry with infinite radius (standard.py:108-111)
  PSF_APER_RADIAL = 1u << 11,// aperture program is a single RADIAL op (fast path)
  PSF_POLY_TRI = 1u << 12,   // bivariate table is triangular (i + j <= rows-1)
};

static inline void mat3_mul(const double* A, const double* B, double* C) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      double s = 0;
      for (int k = 0; k < 3; ++k) s += A[3 * r + k] * B[3 * k + c];
      C[3 * r + c] = s;
    }
}
static inline void mat3_transpose(const double* A, double* At) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) At[3 * c + r] = A[3 * r + c];
}
static inline bool mat3_is_identity(const double* A) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      if (A[3 * r + c] != (r == c ? 1.0 : 0.0)) return false;
  return true;
}

// ---- Zernike -> monomials in (xn, yn) -----------------------------------------
// Z_n^m = R_n^|m|(rho) * {cos(m phi) | sin(|m| phi)},  optiland/zernike/base.py:42-68,
// R_n^m(rho) = sum_k (-1)^k (n-k)! / (k! ((n+m)/2-k)! ((n-m)/2-k)!) rho^(n-2k)  (:217-243)
// rho^j cos(m phi) etc. are polynomials in xn = rho cos(phi), yn = rho sin(phi):
//   rho^(n-2k) {cos|sin}(m phi) = (xn^2+yn^2)^((n-m)/2-k) * {Re|Im} (xn + i yn)^m
static inline double fact(int n) {
  double f = 1;
  for (int i = 2; i <= n; ++i) f *= i;
  return f;
}
static inline double binom(int n, int k) { return fact(n) / (fact(k) * fact(n - k)); }

// Adds coef * Z_n^m to the (deg+1)x(deg+1) row-major table tab[i*(deg+1)+j] ~ xn^i yn^j.
static inline void zernike_add_monomials(int n, int m, double coef, int deg, double* tab) {
  const int ma = m < 0 ? -m : m;
  const int W = deg + 1;
  for (int k = 0; k <= (n - ma) / 2; ++k) {
    double rc = ((k & 1) ? -1.0 : 1.0) * fact(n - k) /
                (fact(k) * fact((n + ma) / 2 - k) * fact((n - ma) / 2 - k));
    const int q = (n - ma) / 2 - k;  // power of (xn^2 + yn^2)
    for (int a = 0; a <= q; ++a) {   // (x^2+y^2)^q = sum_a C(q,a) x^(2a) y^(2(q-a))
      double ca = binom(q, a);
      for (int j = 0; j <= ma; ++j) {  // (x+iy)^m = sum_j C(m,j) x^(m-j) (iy)^j
        // i^j: j%4==0 -> 1, 1 -> i, 2 -> -1, 3 -> -i
        const bool imag = (j & 1) != 0;
        if ((m >= 0) == imag) continue;  // cos wants real part, sin wants imaginary part
        double sgn = ((j >> 1) & 1) ? -1.0 : 1.0;
        int px = 2 * a + (ma - j);
        int py = 2 * (q - a) + j;
        tab[px * W + py] += coef * rc * ca * binom(ma, j) * sgn;
      }
    }
  }
}

// Change of basis a_m -> b_m of the orthonormal polynomials the Q-bfs Clenshaw recurrence runs on
// (G. W. Forbes, Opt. Express 18, 19700 (2010), eqs. A.14-A.16; geometries/forbes/qpoly.py:56-115):
//   f_0 = 2, f_1 = sqrt(19)/2, g_0 = -1/2, h_{n-2} = -n(n-1) / (2 f_{n-2}),
//   g_{n-1} = -(1 + g_{n-2} h_{n-2}) / f_{n-1}, f_n = sqrt(n(n+1) + 3 - g_{n-1}^2 - h_{n-2}^2)
static inline void qbfs_change_basis(const double* a, int nc, std::vector<double>& b) {
  std::vector<double> f(nc + 2), g(nc + 2), h(nc + 2);
  b.assign(nc, 0.0);
  for (int n = 0; n < nc; ++n) {
    if (n == 0) f[0] = 2.0;
    else if (n == 1) { g[0] = -0.5; f[1] = std::sqrt(19.0) / 2.0; }
    else {
      h[n - 2] = -(double)n * (n - 1) / (2.0 * f[n - 2]);
      g[n - 1] = -(1.0 + g[n - 2] * h[n - 2]) / f[n - 1];
      f[n] = std::sqrt((double)n * (n + 1) + 3.0 - g[n - 1] * g[n - 1] - h[n - 2] * h[n - 2]);
    }
  }
  const int m = nc - 1;
  if (m >= 0) b[m] = a[m] / f[m];
  if (m >= 1) b[m - 1] = (a[m - 1] - g[m - 1] * b[m]) / f[m - 1];
  for (int i = m - 2; i >= 0; --i) b[i] = (a[i] - g[i] * b[i + 1] - h[i] * b[i + 2]) / f[i];
}

// Recurrence constants of Forbes' Q-2D polynomials (G. W. Forbes, Opt. Express 20, 2483 (2012); the reference's
// qpoly.py:26-40 and 289-400), in fp64 on the host.  Only the (n, m) the reference evaluates reach them: gamma with
// n >= 1 and m >= 2.
static inline double q2d_gamma(int n, int m) {
  if (n == 1 && m == 2) return 3.0 / 8.0;
  if (n == 1 && m > 2) {
    const int mm1 = m - 1;
    return ((double)(2 * mm1 + 1) / (double)(2 * (mm1 - 1))) * q2d_gamma(1, mm1);
  }
  const int nm1 = n - 1;
  return ((double)((nm1 + 1) * (2 * m + 2 * nm1 - 1)) / (double)((m + nm1 - 2) * (2 * nm1 + 1))) * q2d_gamma(nm1, m);
}
static inline double q2d_dfact(int k) {   // k!! (odd k >= -1)
  double f = 1;
  for (int i = k; i > 1; i -= 2) f *= i;
  return f;
}
static inline double q2d_g_raw(int n, int m) {
  if (n == 0) return q2d_dfact(2 * m - 1) / (std::ldexp(1.0, m + 1) * fact(m - 1));
  if (m == 1) {
    const double t1 = -(double)((2 * n * n - 1) * (n * n - 1)) / (double)(8 * (4 * n * n - 1));
    return t1 - (n == 1 ? 1.0 / 24.0 : 0.0);
  }
  const double num = (double)(2 * n * (m + n - 1) - m) * (double)((n + 1) * (2 * m + 2 * n - 1));
  const double den = (double)((m + 2 * n - 2) * (m + 2 * n - 1)) * (double)((m + 2 * n) * (2 * n + 1));
  return (-num / den) * q2d_gamma(n, m);
}
static inline double q2d_f_raw(int n, int m) {
  if (n == 0 && m == 1) return 0.25;
  if (n == 0) return (double)(m * m) * q2d_dfact(2 * m - 3) / (std::ldexp(1.0, m + 1) * fact(m - 1));
  if (m == 1) {
    const double t1 = (double)(4 * (n - 1) * (n - 1) * n * n + 1) / (double)(8 * (2 * n - 1) * (2 * n - 1));
    return t1 + (n == 1 ? 11.0 / 32.0 : 0.0);
  }
  const int chi = m + n - 2;
  const double num = (double)(2 * n * chi * (3 - 5 * m + 4 * n * chi)) + (double)(m * m * (3 - m + 4 * n * chi));
  const double den = (double)((m + 2 * n - 3) * (m + 2 * n - 2)) * (double)((m + 2 * n - 1) * (2 * n - 1));
  return (num / den) * q2d_gamma(n, m);
}
// f_q2d / g_q2d for n = 0 .. N-1 of one m (the recursion of qpoly.py:340-352 unrolled upwards)
static inline void q2d_fg(int N, int m, std::vector<double>& f, std::vector<double>& g) {
  f.assign(N, 0.0); g.assign(N, 0.0);
  for (int n = 0; n < N; ++n) {
    f[n] = n == 0 ? std::sqrt(q2d_f_raw(0, m)) : std::sqrt(q2d_f_raw(n, m) - g[n - 1] * g[n - 1]);
    g[n] = q2d_g_raw(n, m) / f[n];
  }
}
// abc_q2d_clenshaw(n, m): the reference's special cases (keyed (m, n)), else abc_q2d
static inline void q2d_abc(int n, int m, double& A, double& B, double& C) {
  if (m == 1 && n == 0) { A = 2; B = -1; C = 0; return; }
  if (m == 1 && n == 1) { A = -4.0 / 3.0; B = -8.0 / 3.0; C = -11.0 / 3.0; return; }
  if (m == 1 && n == 2) { A = 9.0 / 5.0; B = -24.0 / 5.0; C = 0; return; }
  if (m == 2 && n == 0) { A = 3; B = -2; C = 0; return; }
  if (m == 3 && n == 0) { A = 5; B = -4; C = 0; return; }
  double d = (double)(4 * n * n - 1) * (double)(m + n - 2) * (double)(m + 2 * n - 3);
  if (d == 0) d = 1e-99;
  const double t1 = (double)((2 * n - 1) * (m + 2 * n - 2)), t2 = (double)(4 * n * (m + n - 2) + (m - 3) * (2 * m - 1));
  A = (t1 * t2) / d;
  B = (double)(-2 * (2 * n - 1) * (m + 2 * n - 3) * (m + 2 * n - 2) * (m + 2 * n - 1)) / d;
  C = (double)(n * (2 * n - 3) * (m + 2 * n - 1) * (2 * m + 2 * n - 3)) / d;
}

enum : uint32_t { HINT_POLY_NEWTON = 1u };   // a polynomial-family / biconic / toroidal Newton surface is present
struct PrepResult {
  std::vector<unsigned char> blob_f64, blob_f32;
  uint32_t features = 0;
  uint32_t hints = 0;          // HINT_* (launch policy only, never semantics)
  bool bwd_supported = true;   // every surface is covered by surface_backward (olb_math.cuh)
  bool bwd_tables = false;     // ... and some surface is a polynomial / Zernike one: its TABLE gradients are wanted
                               // (olb_trace_bwd_* grad_tables)
  int total_gslots = 0;        // per-thread gradient accumulator slots the backward kernel needs
  std::string error;
};

// A polygon of one surface's aperture program: where its prepared instruction sits in the surface's pool, and its
// vertices {x_0, y_0, ...} as uploaded.  The edge block is built per precision (polygon_build), in build_blob.
struct PolygonSource {
  int prog_pos;
  std::vector<double> xy;
};

// Appends the edge block of one polygon to `pool` (whose size is a multiple of 4) and fills in the instruction at
// pool[prog_pos].  Everything is computed in T from the vertices rounded to T, in the reference's operation order.
template <typename T>
static void polygon_build(const std::vector<double>& xy, size_t prog_pos, std::vector<T>& pool) {
  const int n = (int)(xy.size() / 2);
  struct Edge { T vx, vy, vyn, slope; };
  std::vector<Edge> edges;
  T ymin = (T)xy[1], ymax = (T)xy[1];
  for (int e = 0; e < n; ++e) {
    const int j = (e + 1) % n;
    const T vx = (T)xy[2 * e], vy = (T)xy[2 * e + 1], vxn = (T)xy[2 * j], vyn = (T)xy[2 * j + 1];
    if (vy < ymin) ymin = vy;
    if (vy > ymax) ymax = vy;
    if (vy == vyn) continue;              // horizontal: (vy > py) == (vy_next > py) for every py
    const T dx = vxn - vx, dy = vyn - vy;
    edges.push_back({vx, vy, vyn, (T)(dx / dy)});
  }
  int nb = n <= PG_LINEAR_MAX ? 1 : n / PG_PER_BUCKET;
  T scale = 0;
  std::vector<int> b0(edges.size()), b1(edges.size());
  for (;; nb /= 2) {
    scale = nb > 1 ? (T)((T)nb / (T)(ymax - ymin)) : (T)0;
    if (!std::isfinite(scale)) { nb = 1; scale = 0; }
    size_t records = 0;
    for (size_t e = 0; e < edges.size(); ++e) {
      const T lo = edges[e].vy < edges[e].vyn ? edges[e].vy : edges[e].vyn;
      const T hi = edges[e].vy < edges[e].vyn ? edges[e].vyn : edges[e].vy;
      b0[e] = polygon_bucket(lo, ymin, scale, nb);
      b1[e] = polygon_bucket(hi, ymin, scale, nb);
      records += (size_t)(b1[e] - b0[e] + 1);
    }
    if (nb == 1 || records <= 2 * edges.size()) break;
  }
  const size_t block = pool.size();
  pool[prog_pos + PG_NB] = (T)nb;
  pool[prog_pos + PG_YMIN] = ymin;
  pool[prog_pos + PG_YMAX] = ymax;
  pool[prog_pos + PG_SCALE] = scale;
  pool[prog_pos + PG_OFF] = (T)(block - prog_pos);
  pool.resize(block + (size_t)((nb + 1 + 3) & ~3), (T)0);
  int count = 0;
  for (int b = 0; b < nb; ++b) {
    pool[block + b] = (T)count;
    for (size_t e = 0; e < edges.size(); ++e)
      if (b0[e] <= b && b <= b1[e]) {
        pool.push_back(edges[e].vx); pool.push_back(edges[e].vy); pool.push_back(edges[e].vyn); pool.push_back(edges[e].slope);
        ++count;
      }
  }
  pool[block + nb] = (T)count;
}

template <typename T>
static void build_blob(const OlbTable& tab, const std::vector<std::vector<double>>& pools,
                       const std::vector<PrepSurface<double>>& ps, uint32_t features,
                       const std::vector<std::vector<PolygonSource>>& polygons, std::vector<unsigned char>& out) {
  // flatten per-surface pools into one pool, fixing offsets
  std::vector<PrepSurface<T>> surf(ps.size());
  std::vector<T> pool;
  for (size_t s = 0; s < ps.size(); ++s) {
    const PrepSurface<double>& a = ps[s];
    PrepSurface<T>& b = surf[s];
    const int base = (int)pool.size();
    b.kind = a.kind; b.flags = a.flags; b.n_coef = a.n_coef;
    b.coef_off = a.coef_off + base; b.aper_off = a.aper_off + base; b.aper_len = a.aper_len;
    b.max_iter = a.max_iter; b.coating = a.coating; b.media_off = a.media_off + base;
    b.poly_rows = a.poly_rows; b.poly_cols = a.poly_cols; b.poly_d_off = a.poly_d_off + base;
    b.gslot = a.gslot; b.gslots = a.gslots;
    b.phase = a.phase; b.phase_off = a.phase ? a.phase_off + base : 0;
    for (int i = 0; i < 9; ++i) { b.Ag[i] = (T)a.Ag[i]; b.Ar[i] = (T)a.Ar[i]; b.R[i] = (T)a.R[i]; }
    for (int i = 0; i < 3; ++i) { b.bg[i] = (T)a.bg[i]; b.br[i] = (T)a.br[i]; b.t[i] = (T)a.t[i]; }
    b.radius = (T)a.radius; b.curv = (T)a.curv; b.conic = (T)a.conic; b.kp1 = (T)a.kp1;
    b.tol = (T)a.tol; b.coat_t = (T)a.coat_t; b.coat_r = (T)a.coat_r; b.inv_norm = (T)a.inv_norm;
    b.inv_norm_y = (T)a.inv_norm_y; b.curv_y = (T)a.curv_y; b.kp1_y = (T)a.kp1_y; b.r_rot = (T)a.r_rot;
    for (double v : pools[s]) pool.push_back((T)v);
    while (pool.size() % 4) pool.push_back((T)0);
    for (const PolygonSource& pg : polygons[s]) polygon_build<T>(pg.xy, (size_t)base + pg.prog_pos, pool);
  }
  // wavelengths at the end of the pool
  const int wl_off = (int)pool.size();
  for (int j = 0; j < tab.n_wl; ++j) pool.push_back((T)tab.wavelengths[j]);
  while (pool.size() % 4) pool.push_back((T)0);

  PrepHeader h{};
  h.n_surf = (int32_t)ps.size();
  h.n_wl = tab.n_wl;
  h.pool_len = (int32_t)pool.size();
  h.features = features;
  h.elem_size = (int32_t)sizeof(T);
  h.pad[0] = wl_off;
  size_t bytes = sizeof(PrepHeader) + surf.size() * sizeof(PrepSurface<T>) + pool.size() * sizeof(T);
  bytes = (bytes + 15) & ~size_t(15);
  h.blob_bytes = (int32_t)bytes;
  out.assign(bytes, 0);
  unsigned char* p = out.data();
  std::memcpy(p, &h, sizeof(h)); p += sizeof(h);
  std::memcpy(p, surf.data(), surf.size() * sizeof(PrepSurface<T>)); p += surf.size() * sizeof(PrepSurface<T>);
  std::memcpy(p, pool.data(), pool.size() * sizeof(T));
}

static inline int aperture_operands(int op) {
  switch (op) {
    case OLB_AP_RADIAL: return 2;
    case OLB_AP_OFFSET_RADIAL: case OLB_AP_RECT: case OLB_AP_ELLIPSE: return 4;
    case OLB_AP_UNION: case OLB_AP_INTERSECT: case OLB_AP_DIFFERENCE: return 0;
    default: return -1;   // (OLB_AP_POLYGON, of variable length, is handled by the program walk itself)
  }
}

// Validate + prepare. Returns empty error string on success.
static inline PrepResult prepare_table(const OlbTable& tab) {
  PrepResult res;
  if (!tab.surfaces || !tab.wavelengths || !tab.pool) { res.error = "NULL table member"; return res; }
  if (tab.n_surfaces < 1 || tab.n_surfaces > OLB_MAX_SURFACES) { res.error = "n_surfaces out of range"; return res; }
  if (tab.n_wl < 1 || tab.n_wl > OLB_MAX_WAVELENGTHS) { res.error = "n_wl out of range"; return res; }
  const int n_wl = tab.n_wl;
  std::vector<PrepSurface<double>> ps(tab.n_surfaces);
  std::vector<std::vector<double>> pools(tab.n_surfaces);
  uint32_t features = 0;
  int prev = -1;  // previous surface with a frame (non-NOOP)
  int64_t grid_elements = 0, polygon_vertices = 0, q2d_elements = 0;
  std::vector<std::vector<PolygonSource>> polygons(tab.n_surfaces);
  auto in_pool = [&](int off, int len) { return off >= 0 && len >= 0 && (int64_t)off + len <= tab.pool_len; };

  for (int s = 0; s < tab.n_surfaces; ++s) {
    const OlbSurface& in = tab.surfaces[s];
    PrepSurface<double>& o = ps[s];
    std::memset(&o, 0, sizeof(o));
    std::vector<double>& pool = pools[s];
    o.kind = in.kind;
    o.flags = in.flags & 0xffu;
    o.max_iter = in.max_iter;
    o.coating = in.coating;
    if (in.kind < OLB_GEOM_NOOP || in.kind > OLB_GEOM_FORBES_Q2D) { res.error = "unknown geometry kind"; return res; }

    // ---- pose --------------------------------------------------------------
    if (in.kind != OLB_GEOM_NOOP) {
      bool finite = std::isfinite(in.t[0]) && std::isfinite(in.t[1]) && std::isfinite(in.t[2]);
      for (int i = 0; i < 9; ++i) finite = finite && std::isfinite(in.R[i]);
      if (!finite) { res.error = "non-finite surface pose"; return res; }
    }
    double Rt[9];
    mat3_transpose(in.R, Rt);
    for (int i = 0; i < 9; ++i) { o.R[i] = in.R[i]; o.Ag[i] = Rt[i]; }
    for (int i = 0; i < 3; ++i) o.t[i] = in.t[i];
    const bool rotated = !mat3_is_identity(in.R);
    for (int r = 0; r < 3; ++r) {
      if (rotated) o.bg[r] = -(Rt[3 * r] * in.t[0] + Rt[3 * r + 1] * in.t[1] + Rt[3 * r + 2] * in.t[2]);
      else o.bg[r] = -in.t[r];
    }
    if (rotated) { o.flags |= OLB_SF_ROTATED | PSF_ROT_IN_G; features |= FEAT_ROT; }
    else o.flags &= ~uint32_t(OLB_SF_ROTATED);
    if (in.kind != OLB_GEOM_NOOP) {
      if (prev >= 0) {
        const OlbSurface& pv = tab.surfaces[prev];
        const bool prev_rot = !mat3_is_identity(pv.R);
        if (!rotated && !prev_rot) {
          for (int i = 0; i < 9; ++i) o.Ar[i] = (i % 4 == 0) ? 1.0 : 0.0;
          for (int r = 0; r < 3; ++r) o.br[r] = pv.t[r] - in.t[r];
        } else {
          mat3_mul(Rt, pv.R, o.Ar);  // R_cur^T R_prev
          double d[3] = {pv.t[0] - in.t[0], pv.t[1] - in.t[1], pv.t[2] - in.t[2]};
          for (int r = 0; r < 3; ++r) o.br[r] = Rt[3 * r] * d[0] + Rt[3 * r + 1] * d[1] + Rt[3 * r + 2] * d[2];
          if (!mat3_is_identity(o.Ar)) { o.flags |= PSF_ROT_IN_R; features |= FEAT_ROT; }
        }
      } else {
        for (int i = 0; i < 9; ++i) o.Ar[i] = o.Ag[i];
        for (int r = 0; r < 3; ++r) o.br[r] = o.bg[r];
        if (rotated) o.flags |= PSF_ROT_IN_R;
      }
      prev = s;
    }

    // ---- geometry ----------------------------------------------------------
    o.radius = in.radius; o.conic = in.conic; o.kp1 = 1.0 + in.conic;
    o.tol = in.tol;
    o.coat_t = in.coat_t; o.coat_r = in.coat_r;
    o.inv_norm = 1.0; o.inv_norm_y = 1.0; o.curv_y = 0; o.kp1_y = 1.0; o.r_rot = INFINITY;
    if (in.kind == OLB_GEOM_PLANE || in.kind == OLB_GEOM_NOOP) { o.radius = INFINITY; o.curv = 0; }
    else if (std::isinf(in.radius)) { o.curv = 0; o.flags |= PSF_RADIUS_INF; }
    else { o.curv = 1.0 / in.radius; }
    const bool newton = in.kind >= OLB_GEOM_EVEN_ASPHERE && in.kind != OLB_GEOM_GRID_SAG;
    if (in.kind == OLB_GEOM_GRID_SAG) {
      // x[nx], y[ny], sag[ny][nx] as they are: the kernel's cell search and interpolation are the reference's
      const int nx = in.aux0, ny = in.n_coef;
      if (nx < 2 || ny < 2) { res.error = "grid sag: nx and ny must be >= 2"; return res; }
      const int64_t elems = (int64_t)nx + ny + (int64_t)nx * ny;
      grid_elements += elems;
      if (grid_elements > OLB_MAX_GRID_ELEMENTS) {
        res.error = "grid sag: the grids of this table exceed " + std::to_string(OLB_MAX_GRID_ELEMENTS) +
                    " prepared elements (they are staged in shared memory)";
        return res;
      }
      if (!in_pool(in.coef_off, (int)elems)) { res.error = "grid sag block outside pool"; return res; }
      const double* g = tab.pool + in.coef_off;
      for (int a = 0; a < 2; ++a) {
        const double* c = a == 0 ? g : g + nx;
        const int n = a == 0 ? nx : ny;
        for (int k = 0; k < n; ++k)
          if (!std::isfinite(c[k]) || (k > 0 && !(c[k] > c[k - 1]))) {
            res.error = "grid sag: coordinates must be finite and strictly increasing"; return res;
          }
      }
      for (int64_t k = nx + ny; k < elems; ++k)
        if (!std::isfinite(g[k])) { res.error = "grid sag: non-finite sag value"; return res; }
      if (in.max_iter < 0) { res.error = "negative max_iter"; return res; }
      o.radius = INFINITY; o.curv = 0; o.conic = 0; o.kp1 = 1.0;
      o.poly_cols = nx; o.poly_rows = ny;
      o.coef_off = (int)pool.size();
      pool.insert(pool.end(), g, g + elems);
      while (pool.size() % 4) pool.push_back(0);
      features |= FEAT_GRID;
    }
    if (newton) {
      features |= FEAT_NEWTON;
      if (in.kind != OLB_GEOM_EVEN_ASPHERE && in.kind != OLB_GEOM_ODD_ASPHERE) { res.hints |= HINT_POLY_NEWTON; features |= FEAT_FREEFORM; }
      if (in.max_iter < 0) { res.error = "negative max_iter"; return res; }
    }
    if (in.kind == OLB_GEOM_EVEN_ASPHERE || in.kind == OLB_GEOM_ODD_ASPHERE) {
      if (!in_pool(in.coef_off, in.n_coef)) { res.error = "coefficient block outside pool"; return res; }
      o.n_coef = in.n_coef;
      o.coef_off = (int)pool.size();
      for (int i = 0; i < in.n_coef; ++i) pool.push_back(tab.pool[in.coef_off + i]);
      while (pool.size() % 4) pool.push_back(0);
      // slope coefficients, so that the Newton loop does one FMA per term: 2(i+1) C_i (even), (i+1) C_i (odd)
      o.poly_d_off = (int)pool.size();
      const double step = in.kind == OLB_GEOM_EVEN_ASPHERE ? 2.0 : 1.0;
      for (int i = 0; i < in.n_coef; ++i) pool.push_back(step * (i + 1) * tab.pool[in.coef_off + i]);
      while (pool.size() % 4) pool.push_back(0);
    } else if (in.kind == OLB_GEOM_POLYNOMIAL) {
      const int cols = in.aux0 > 0 ? in.aux0 : 1;
      if (in.n_coef % cols || !in_pool(in.coef_off, in.n_coef)) { res.error = "bad polynomial block"; return res; }
      o.poly_rows = in.n_coef / cols; o.poly_cols = cols;
      if (o.poly_rows > 24 || cols > 24) { res.error = "polynomial order too high (max 23)"; return res; }
      o.coef_off = (int)pool.size();
      for (int i = 0; i < in.n_coef; ++i) pool.push_back(tab.pool[in.coef_off + i]);
      while (pool.size() % 4) pool.push_back(0);
      o.poly_d_off = o.coef_off;  // derivative of the same polynomial (polynomial.py:123-155)
      o.inv_norm = 1.0;
    } else if (in.kind == OLB_GEOM_CHEBYSHEV) {
      // conic + sum C_ij T_i(x/nx) T_j(y/ny)  (chebyshev.py:126-150): expanded into monomials of
      // (xn, yn) with the integer coefficients of T_n (T_0 = 1, T_1 = x, T_{n+1} = 2x T_n - T_{n-1}).
      const int cols = in.aux0 > 0 ? in.aux0 : 1;
      if (in.n_coef % cols || !in_pool(in.coef_off, in.n_coef + 2)) { res.error = "bad Chebyshev block"; return res; }
      const int rows = in.n_coef / cols;
      if (rows > 24 || cols > 24) { res.error = "Chebyshev order too high (max 23)"; return res; }
      const double nx = tab.pool[in.coef_off], ny = tab.pool[in.coef_off + 1];
      if (!(nx > 0) || !(ny > 0)) { res.error = "Chebyshev norms must be positive"; return res; }
      const int M = rows > cols ? rows : cols;
      std::vector<std::vector<double>> Tc(M, std::vector<double>(M, 0.0));  // Tc[n][p]: coefficient of x^p in T_n
      Tc[0][0] = 1.0;
      if (M > 1) Tc[1][1] = 1.0;
      for (int n = 2; n < M; ++n)
        for (int p = 0; p < M; ++p) Tc[n][p] = (p > 0 ? 2.0 * Tc[n - 1][p - 1] : 0.0) - Tc[n - 2][p];
      std::vector<double> Pm(rows * cols, 0.0);
      for (int i = 0; i < rows; ++i)
        for (int j = 0; j < cols; ++j) {
          const double c = tab.pool[in.coef_off + 2 + i * cols + j];
          if (c == 0) continue;
          for (int p = 0; p <= i; ++p)
            for (int q = 0; q <= j; ++q) Pm[p * cols + q] += c * Tc[i][p] * Tc[j][q];
        }
      o.poly_rows = rows; o.poly_cols = cols;
      o.coef_off = (int)pool.size();
      pool.insert(pool.end(), Pm.begin(), Pm.end());
      while (pool.size() % 4) pool.push_back(0);
      o.poly_d_off = o.coef_off;
      o.inv_norm = 1.0 / nx; o.inv_norm_y = 1.0 / ny;
    } else if (in.kind == OLB_GEOM_BICONIC) {
      if (!in_pool(in.coef_off, 2)) { res.error = "biconic block outside pool"; return res; }
      const double Ry = tab.pool[in.coef_off], ky = tab.pool[in.coef_off + 1];
      // cx / cy = 0 for an infinite or zero radius (biconic.py:63-64)
      if (std::isinf(in.radius) || in.radius == 0) o.curv = 0;
      o.curv_y = (std::isinf(Ry) || Ry == 0) ? 0.0 : 1.0 / Ry;
      o.kp1_y = 1.0 + ky;
    } else if (in.kind == OLB_GEOM_TOROIDAL) {
      if (!in_pool(in.coef_off, 2 + in.n_coef) || in.n_coef < 0) { res.error = "toroidal block outside pool"; return res; }
      if (in.conic != 0) { res.error = "toroidal: OlbSurface.conic must be 0 (the Newton start sphere)"; return res; }
      o.r_rot = tab.pool[in.coef_off];
      o.kp1_y = 1.0 + tab.pool[in.coef_off + 1];
      o.curv_y = (std::isfinite(in.radius) && in.radius != 0) ? 1.0 / in.radius : 0.0;  // c_yz (toroidal.py:82-84)
      o.n_coef = in.n_coef;
      o.coef_off = (int)pool.size();
      for (int i = 0; i < in.n_coef; ++i) pool.push_back(tab.pool[in.coef_off + 2 + i]);
      while (pool.size() % 4) pool.push_back(0);
    } else if (in.kind == OLB_GEOM_FORBES_QBFS) {
      if (in.n_coef < 0 || in.n_coef > 64 || !in_pool(in.coef_off, in.n_coef)) { res.error = "bad Forbes coefficient block"; return res; }
      if (!(in.norm_radius > 0)) { res.error = "Forbes norm_radius must be positive"; return res; }
      const int nc = in.n_coef;
      const double* a = tab.pool + in.coef_off;
      std::vector<double> b;
      qbfs_change_basis(a, nc, b);
      bool all_zero = true;
      for (int i = 0; i < nc; ++i) all_zero = all_zero && a[i] == 0.0;
      o.n_coef = all_zero ? 0 : nc;    // no / all-zero terms: the reference's slope takes the base-conic branch
      o.coef_off = (int)pool.size();
      for (int i = 0; i < nc; ++i) pool.push_back(b[i]);
      while (pool.size() % 4) pool.push_back(0);
      o.inv_norm = 1.0 / in.norm_radius;
      features |= FEAT_EXTRA;          // the Forbes code lives in the general kernel only (olb_math.cuh::newton_sag)
    } else if (in.kind == OLB_GEOM_FORBES_Q2D) {
      // cm0[n0], {na_m, nb_m} x M, then the lists (include/olb.h "Forbes Q-2D")
      const int n0 = in.aux0, M = in.n_coef;
      if (M < 0 || M > OLB_Q2D_MAX_M) { res.error = "Forbes Q-2D: M out of range (max " + std::to_string(OLB_Q2D_MAX_M) + ")"; return res; }
      if (n0 < 0 || n0 > OLB_Q2D_MAX_TERMS || !in_pool(in.coef_off, n0 + 2 * M)) { res.error = "bad Forbes Q-2D block"; return res; }
      if (!(in.norm_radius > 0) || !std::isfinite(in.norm_radius)) { res.error = "Forbes Q-2D norm_radius must be positive and finite"; return res; }
      const double* blk = tab.pool + in.coef_off;
      std::vector<int> na(M), nb(M);
      int len = n0 + 2 * M;
      int64_t elems = Q2_HDR + n0;
      for (int m = 0; m < M; ++m) {
        const double da = blk[n0 + 2 * m], db = blk[n0 + 2 * m + 1];
        if (!(da >= 0 && da <= OLB_Q2D_MAX_TERMS && da == std::floor(da)) || !(db >= 0 && db <= OLB_Q2D_MAX_TERMS && db == std::floor(db))) {
          res.error = "Forbes Q-2D: list lengths must be integers in [0, " + std::to_string(OLB_Q2D_MAX_TERMS) + "]"; return res;
        }
        na[m] = (int)da; nb[m] = (int)db;
        len += na[m] + nb[m];
        elems += Q2_MHDR + 3 * std::max(na[m], nb[m]) + na[m] + nb[m];
      }
      if (!in_pool(in.coef_off, len)) { res.error = "Forbes Q-2D block outside pool"; return res; }
      for (int k = 0; k < len; ++k)
        if (!std::isfinite(blk[k])) { res.error = "Forbes Q-2D: non-finite coefficient"; return res; }
      q2d_elements += elems;
      if (q2d_elements > OLB_MAX_Q2D_ELEMENTS) {
        res.error = "Forbes Q-2D: the surfaces of this table exceed " + std::to_string(OLB_MAX_Q2D_ELEMENTS) +
                    " prepared elements (they are staged in shared memory)";
        return res;
      }
      while (pool.size() % 4) pool.push_back(0);
      o.coef_off = (int)pool.size();
      o.n_coef = M; o.poly_rows = n0;
      o.inv_norm = 1.0 / in.norm_radius;
      pool.insert(pool.end(), Q2_HDR, 0.0);
      pool[o.coef_off + Q2_NORM] = in.norm_radius;
      std::vector<double> b;
      qbfs_change_basis(blk, n0, b);                 // m = 0: compute_z_zprime_qbfs (qpoly.py:265-283)
      pool.insert(pool.end(), b.begin(), b.end());
      const double* lists = blk + n0 + 2 * M;
      for (int m = 1; m <= M; ++m) {
        const int N = std::max(na[m - 1], nb[m - 1]);
        std::vector<double> f, g;
        q2d_fg(N, m, f, g);
        pool.push_back(na[m - 1]); pool.push_back(nb[m - 1]); pool.push_back(N); pool.push_back(0);
        const size_t abc = pool.size();
        for (int n = 0; n < N; ++n) {
          double A, B, C, A1, B1, C1;
          q2d_abc(n, m, A, B, C);
          q2d_abc(n + 1, m, A1, B1, C1);
          pool.push_back(A); pool.push_back(B); pool.push_back(C1);
        }
        for (int side = 0; side < 2; ++side) {
          const int nl = side == 0 ? na[m - 1] : nb[m - 1];
          const double* c = lists;
          lists += nl;
          // change_basis_q2d_to_pnm (qpoly.py:355-370)
          std::vector<double> d(nl);
          for (int n = nl - 1; n >= 0; --n) d[n] = n == nl - 1 ? c[n] / f[n] : (c[n] - g[n] * d[n + 1]) / f[n];
          if (m == 1 && nl > 0) {
            // vertex slope (geometry.py:596-609): the m = 1 sum at usq = 0, divided by norm_radius
            double a1 = 0, a2 = 0, a0 = 0, a3 = 0;
            for (int n = nl - 1; n >= 0; --n) {
              a0 = d[n] + pool[abc + 3 * n] * a1 - pool[abc + 3 * n + 2] * a2;
              if (n == 3) a3 = a0;
              a2 = a1; a1 = a0;
            }
            pool[o.coef_off + (side == 0 ? Q2_VX : Q2_VY)] = (0.5 * a0 - (nl > 3 ? 2.0 / 5.0 * a3 : 0.0)) / in.norm_radius;
          }
          pool.insert(pool.end(), d.begin(), d.end());
        }
      }
      while (pool.size() % 4) pool.push_back(0);
      features |= FEAT_EXTRA | FEAT_Q2D;
    } else if (in.kind == OLB_GEOM_ZERNIKE) {
      if (!in_pool(in.coef_off, 4 * in.n_coef)) { res.error = "Zernike block outside pool"; return res; }
      if (!(in.norm_radius > 0)) { res.error = "Zernike norm_radius must be positive"; return res; }
      int deg = 0;
      for (int i = 0; i < in.n_coef; ++i) {
        const double* tm = tab.pool + in.coef_off + 4 * i;
        int n = (int)tm[0], m = (int)tm[1];
        if (n < 0 || (m < 0 ? -m : m) > n || ((n - m) & 1) || n > 23) { res.error = "bad Zernike (n, m)"; return res; }
        if (n > deg) deg = n;
      }
      // table width padded to one of the compile-time sizes of olb_math.cuh::poly_tri_value (zero rows / columns:
      // the nested Horner is unchanged); wider tables run the runtime-sized loops
      int degp = deg;
      for (int wp : {4, 8, 12})
        if (deg + 1 <= wp) { degp = wp - 1; break; }
      const int W = degp + 1;
      std::vector<double> S(W * W, 0.0), D(W * W, 0.0);
      for (int i = 0; i < in.n_coef; ++i) {
        const double* tm = tab.pool + in.coef_off + 4 * i;
        zernike_add_monomials((int)tm[0], (int)tm[1], tm[2], degp, S.data());  // c * N_nm
        zernike_add_monomials((int)tm[0], (int)tm[1], tm[3], degp, D.data());  // c (quirk: no N_nm)
      }
      o.poly_rows = W; o.poly_cols = W; o.flags |= PSF_POLY_TRI;
      while (pool.size() % 4) pool.push_back(0);     // 16-byte aligned rows: the kernel loads them as vectors
      o.coef_off = (int)pool.size();
      pool.insert(pool.end(), S.begin(), S.end());
      while (pool.size() % 4) pool.push_back(0);
      o.poly_d_off = (int)pool.size();
      pool.insert(pool.end(), D.begin(), D.end());
      while (pool.size() % 4) pool.push_back(0);
      o.inv_norm = 1.0 / in.norm_radius; o.inv_norm_y = o.inv_norm;
    }

    // ---- aperture ------------------------------------------------------------
    if (in.flags & OLB_SF_APERTURE) {
      if (!in_pool(in.aper_off, in.aper_len) || in.aper_len < 1) { res.error = "aperture program outside pool"; return res; }
      int i = 0, depth = 0;
      o.aper_off = (int)pool.size();
      while (i < in.aper_len) {
        int op = (int)tab.pool[in.aper_off + i];
        int nops = aperture_operands(op);
        if (op == OLB_AP_POLYGON) {
          // {opcode, n, x_0, y_0, ...} -> the prepared instruction (PG_*), completed per precision in build_blob
          const double nd = i + 1 < in.aper_len ? tab.pool[in.aper_off + i + 1] : 0.0;
          if (!(nd >= 3 && nd <= OLB_MAX_POLYGON_VERTICES && nd == (double)(int)nd)) {
            res.error = "polygon aperture: the vertex count must be an integer in [3, " + std::to_string(OLB_MAX_POLYGON_VERTICES) + "]";
            return res;
          }
          nops = 1 + 2 * (int)nd;
          if (i + 1 + nops > in.aper_len) { res.error = "polygon aperture: vertices outside the program"; return res; }
          polygon_vertices += (int)nd;
          if (polygon_vertices > OLB_MAX_POLYGON_VERTICES) {
            res.error = "polygon aperture: the polygons of this table have more than " + std::to_string(OLB_MAX_POLYGON_VERTICES) +
                        " vertices (their edges are staged in shared memory)";
            return res;
          }
          const double* xy = tab.pool + in.aper_off + i + 2;
          for (int k = 0; k < 2 * (int)nd; ++k)
            if (!std::isfinite(xy[k])) { res.error = "polygon aperture: non-finite vertex"; return res; }
          polygons[s].push_back({(int)pool.size(), std::vector<double>(xy, xy + 2 * (int)nd)});
          pool.push_back((double)op);
          pool.insert(pool.end(), PG_LEN - 1, 0.0);
          features |= FEAT_POLYGON;
        } else {
          if (nops < 0) { res.error = "bad aperture opcode"; return res; }
          for (int k = 0; k <= nops; ++k) pool.push_back(i + k < in.aper_len ? tab.pool[in.aper_off + i + k] : 0.0);
        }
        if (op >= OLB_AP_UNION) { if (depth < 2) { res.error = "aperture stack underflow"; return res; } depth -= 1; }
        else { depth += 1; if (depth > 8) { res.error = "aperture program too deep"; return res; } }
        i += 1 + nops;
      }
      if (i != in.aper_len || depth != 1) { res.error = "malformed aperture program"; return res; }
      o.aper_len = (int)pool.size() - o.aper_off;
      while (pool.size() % 4) pool.push_back(0);
      if ((int)tab.pool[in.aper_off] == OLB_AP_RADIAL && in.aper_len == 3) {
        o.flags |= PSF_APER_RADIAL;
        // store squared radii right after the program for the fast path
        double rmax = tab.pool[in.aper_off + 1], rmin = tab.pool[in.aper_off + 2];
        pool[o.aper_off + 1] = rmax * rmax;  // reference compares r2 <= r_max**2 (radial.py:68-69)
        pool[o.aper_off + 2] = rmin * rmin;
      } else {
        features |= FEAT_EXTRA;
      }
    }

    // ---- media -----------------------------------------------------------------
    if (!in_pool(in.media_off, 5 * n_wl)) { res.error = "media block outside pool"; return res; }

    // ---- BSDF block {kind, sigma, seed_lo, seed_hi} at media_off + 5 n_wl (include/olb.h) -----------------------
    const bool bsdf = (in.flags & OLB_SF_BSDF) != 0;
    double bsdf_block[BS_LEN] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (bsdf) {
      if (in.kind == OLB_GEOM_NOOP) { res.error = "BSDF on an object surface"; return res; }
      const int bb = in.media_off + 5 * n_wl;
      if (!in_pool(bb, 4)) { res.error = "BSDF block outside pool"; return res; }
      const double* b = tab.pool + bb;
      if (b[0] != OLB_BSDF_LAMBERTIAN && b[0] != OLB_BSDF_GAUSSIAN) { res.error = "bad BSDF block: unknown kind"; return res; }
      if (!std::isfinite(b[1])) { res.error = "bad BSDF block: non-finite sigma"; return res; }
      for (int q = 2; q < 4; ++q)
        if (!(b[q] >= 0 && b[q] < 4294967296.0 && b[q] == std::floor(b[q]))) {
          res.error = "bad BSDF block: the seed halves must be integers in [0, 2^32)"; return res;
        }
      const uint64_t key = (uint64_t)b[2] | ((uint64_t)b[3] << 32);
      bsdf_block[BS_KIND] = b[0];
      bsdf_block[BS_SIGMA] = b[1];
      for (int q = 0; q < 4; ++q) bsdf_block[BS_KEY + q] = (double)((key >> (16 * q)) & 0xffffu);
      features |= FEAT_BSDF;
      res.bwd_supported = false;       // the adjoint has no scatter
    }

    // ---- thin-film / polarizer / retarder coating: its prepared block goes right before the media block ------
    if (in.coating >= OLB_COAT_THIN_FILM && in.coating <= OLB_COAT_RETARDER) {
      if (in.kind == OLB_GEOM_NOOP) { res.error = "polarizing coating on an object surface"; return res; }
      const int cb = in.media_off + 5 * n_wl + (bsdf ? 4 : 0);
      std::vector<double> hdr(CO_HDR, 0.0);
      if (in.coating == OLB_COAT_THIN_FILM) {
        if (!in_pool(cb, 1)) { res.error = "thin-film block outside pool"; return res; }
        const double Ld = tab.pool[cb];
        const int L = (int)Ld;
        if (!(Ld == (double)L) || L < 0 || L > OLB_MAX_FILM_LAYERS) {
          res.error = "bad thin-film block: number of layers out of range"; return res;
        }
        if (!in_pool(cb, 1 + L + n_wl * (4 + 2 * L))) { res.error = "thin-film block outside pool"; return res; }
        const double* d = tab.pool + cb + 1;
        for (int l = 0; l < L; ++l)
          if (!std::isfinite(d[l]) || d[l] < 0) { res.error = "bad thin-film block: thickness not finite and >= 0"; return res; }
        int stride = CO_REC + CO_LAYER * L;
        while (stride % 4) ++stride;
        for (int j = 0; j < n_wl; ++j) {
          const double* w = tab.pool + cb + 1 + L + j * (4 + 2 * L);
          const size_t r0 = pool.size();
          pool.push_back(w[0] * w[0] - w[1] * w[1]);   // incident n0~^2 = A0 + i B0
          pool.push_back(2.0 * w[0] * w[1]);
          pool.push_back(w[2] * w[2] - w[3] * w[3]);   // substrate
          pool.push_back(2.0 * w[2] * w[3]);
          const double k0 = 2.0 / tab.wavelengths[j];     // phase thickness / pi per unit sqrt(X) and thickness
          for (int l = 0; l < L; ++l) {
            const double n = w[4 + 2 * l], k = w[5 + 2 * l];
            const double A = n * n - k * k, B = 2.0 * n * k;
            const double m2 = FILM_Y * (A * A + B * B);   // 1 / (Y (A - iB)) = (A + iB) / (Y (A^2 + B^2))
            pool.push_back(k0 * d[l]);
            pool.push_back(A);
            pool.push_back(B);
            pool.push_back(A / m2);
            pool.push_back(B / m2);
          }
          while (pool.size() - r0 < (size_t)stride) pool.push_back(0);
        }
        hdr[CO_L] = L;
        hdr[CO_STRIDE] = stride;
        hdr[CO_BACK] = (double)stride * n_wl;
      } else {
        const int na = in.coating == OLB_COAT_POLARIZER ? 3 : 4;
        if (!in_pool(cb, na)) { res.error = "polarizer / retarder block outside pool"; return res; }
        const double* a = tab.pool + cb + (na - 3);
        const double norm = std::sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
        if (!std::isfinite(norm) || norm == 0) { res.error = "bad polarizer / retarder block: axis not finite and non-zero"; return res; }
        for (int q = 0; q < 3; ++q) hdr[CO_AX + q] = a[q];
        if (in.coating == OLB_COAT_RETARDER) {
          const double dr = tab.pool[cb];
          if (!std::isfinite(dr)) { res.error = "bad retarder block: non-finite retardance"; return res; }
          hdr[CO_COS] = std::cos(dr / 2);
          hdr[CO_SIN] = std::sin(dr / 2);
        }
      }
      pool.insert(pool.end(), hdr.begin(), hdr.end());
      features |= FEAT_POL | FEAT_JONES;
      res.bwd_supported = false;       // the adjoint has no polarization
    }
    if (bsdf) pool.insert(pool.end(), bsdf_block, bsdf_block + BS_LEN);
    o.media_off = (int)pool.size();
    bool absorbing = false;
    for (int j = 0; j < n_wl; ++j) {
      const double n1 = tab.pool[in.media_off + 0 * n_wl + j];
      const double n2 = tab.pool[in.media_off + 1 * n_wl + j];
      const double k1 = tab.pool[in.media_off + 2 * n_wl + j];
      const double c1 = tab.pool[in.media_off + 3 * n_wl + j];
      const double c2 = tab.pool[in.media_off + 4 * n_wl + j];
      if (k1 > 0) absorbing = true;
      pool.push_back(n1);
      pool.push_back(n1 / n2);
      pool.push_back(4.0 * M_PI * k1 / tab.wavelengths[j] * 1e3);
      pool.push_back(c2 / c1);
    }
    if (absorbing) o.flags |= OLB_SF_ABSORBING;
    else o.flags &= ~uint32_t(OLB_SF_ABSORBING);
    if (in.coating == OLB_COAT_SIMPLE) features |= FEAT_EXTRA;
    else if (in.coating == OLB_COAT_FRESNEL) features |= FEAT_POL;
    else if (in.coating != OLB_COAT_NONE && !(in.coating >= OLB_COAT_THIN_FILM && in.coating <= OLB_COAT_RETARDER)) {
      res.error = "unknown coating"; return res;
    }

    // ---- ruled grating (DiffractiveInteractionModel) ---------------------------------------------
    if (in.interaction == OLB_INTERACT_GRATING) {
      if (in.kind == OLB_GEOM_NOOP) { res.error = "grating interaction on an object surface"; return res; }
      if (in.kind != OLB_GEOM_PLANE && in.kind != OLB_GEOM_STANDARD) {
        res.error = "grating interaction on a geometry other than a plane or a conic"; return res;
      }
      if (in.kind == OLB_GEOM_STANDARD && !std::isfinite(in.radius)) {
        res.error = "grating interaction on a conic with an infinite radius"; return res;
      }
      if (!in_pool(in.phase_off, 5)) { res.error = "grating block outside pool"; return res; }
      const double* gb = tab.pool + in.phase_off;
      if (!(gb[1] == 3.0)) { res.error = "bad grating block: wrong number of terms"; return res; }
      if (!(gb[0] == 1.0)) { res.error = "bad grating block: efficiency must be exactly 1"; return res; }
      const double m = gb[2], d = gb[3], alpha = gb[4];
      if (!std::isfinite(m) || !std::isfinite(alpha)) { res.error = "bad grating block: non-finite order or angle"; return res; }
      if (!std::isfinite(d) || d == 0) { res.error = "bad grating block: non-finite or zero period"; return res; }
      o.phase = in.interaction;
      o.phase_off = (int)pool.size();
      pool.push_back(1.0);
      pool.push_back(3.0);
      pool.push_back(std::sin(alpha));
      pool.push_back(std::cos(alpha));
      pool.push_back(std::tan(alpha));
      pool.push_back(d > 0 ? 1.0 : -1.0);
      for (int j = 0; j < n_wl; ++j) {
        pool.push_back(m * tab.wavelengths[j] / d);
        pool.push_back(tab.pool[in.media_off + n_wl + j]);
      }
      while (pool.size() % 4) pool.push_back(0);
      features |= FEAT_GRATING;
      res.bwd_supported = false;       // the adjoint has no grating interaction
    } else if (in.interaction != OLB_INTERACT_REFRACT) {
      // ---- phase-profile interaction (PhaseInteractionModel) -------------------------------------
      if (in.interaction < OLB_INTERACT_PHASE_CONSTANT || in.interaction > OLB_INTERACT_PHASE_RADIAL) {
        res.error = "unknown interaction model"; return res;
      }
      if (in.kind == OLB_GEOM_NOOP) { res.error = "phase interaction on an object surface"; return res; }
      if (!in_pool(in.phase_off, 2)) { res.error = "phase block outside pool"; return res; }
      const double eff = tab.pool[in.phase_off], ntd = tab.pool[in.phase_off + 1];
      const int nt = (int)ntd;
      const int want = in.interaction == OLB_INTERACT_PHASE_CONSTANT ? 1 : in.interaction == OLB_INTERACT_PHASE_LINEAR ? 2 : -1;
      if (!(ntd == (double)nt) || (want > 0 && nt != want) || (want < 0 && (nt < 1 || nt > OLB_MAX_PHASE_TERMS))) {
        res.error = "bad phase block: wrong number of profile terms"; return res;
      }
      if (!in_pool(in.phase_off, 2 + nt)) { res.error = "phase block outside pool"; return res; }
      if (!std::isfinite(eff)) { res.error = "bad phase block: non-finite efficiency"; return res; }
      const double* prm = tab.pool + in.phase_off + 2;
      o.phase = in.interaction;
      o.phase_off = (int)pool.size();
      pool.push_back(eff);
      pool.push_back((double)nt);
      for (int p = 0; p < nt; ++p) pool.push_back(prm[p]);
      if (in.interaction == OLB_INTERACT_PHASE_RADIAL)
        for (int p = 0; p < nt; ++p) pool.push_back(2.0 * (p + 1) * prm[p]);
      for (int j = 0; j < n_wl; ++j) {
        pool.push_back(tab.wavelengths[j] * 1e-3 / (2.0 * M_PI));
        pool.push_back((in.flags & OLB_SF_REFLECT) ? tab.pool[in.media_off + j] : tab.pool[in.media_off + n_wl + j]);
      }
      while (pool.size() % 4) pool.push_back(0);
      features |= FEAT_PHASE;
      res.bwd_supported = false;       // the adjoint has no phase interaction
    }
  }
  res.features = features;
  int gslot = 0;
  for (int s = 0; s < tab.n_surfaces; ++s) {
    ps[s].gslot = gslot;
    // 7 scalars + even-asphere coefficients + (tilted pose) the 9 entries of dLoss/dR
    // (a Forbes Q^bfs surface carries the gradients of its Clenshaw-basis coefficients in the same slots)
    const bool asph = ps[s].kind == OLB_GEOM_EVEN_ASPHERE || ps[s].kind == OLB_GEOM_ODD_ASPHERE ||
                      ps[s].kind == OLB_GEOM_FORBES_QBFS;
    ps[s].gslots = ps[s].kind == OLB_GEOM_NOOP ? 0 : 7 + (asph ? ps[s].n_coef : 0) +
                                                         ((ps[s].flags & OLB_SF_ROTATED) ? 9 : 0);
    gslot += ps[s].gslots;
  }
  res.total_gslots = gslot;
  for (int s = 0; s < tab.n_surfaces; ++s) {
    const PrepSurface<double>& o = ps[s];
    const bool polyfam = (o.kind == OLB_GEOM_POLYNOMIAL || o.kind == OLB_GEOM_ZERNIKE || o.kind == OLB_GEOM_CHEBYSHEV) &&
                         o.poly_rows <= 12 && o.poly_cols <= 12;
    const bool kind_ok = o.kind == OLB_GEOM_NOOP || o.kind == OLB_GEOM_PLANE || o.kind == OLB_GEOM_STANDARD ||
                         ((o.kind == OLB_GEOM_EVEN_ASPHERE || o.kind == OLB_GEOM_ODD_ASPHERE) && o.n_coef <= 12) || polyfam;
    // Forbes Q^bfs: covered by the general (grad_tables) variant of the adjoint kernel, at most 12 terms
    const bool forbes = o.kind == OLB_GEOM_FORBES_QBFS && tab.surfaces[s].n_coef <= 12;
    // grid sag: covered by the same variant (its branch lives there, so the lean variant keeps its code)
    const bool grid = o.kind == OLB_GEOM_GRID_SAG;
    if (polyfam || forbes || grid) res.bwd_tables = true;
    if (features & FEAT_POLYGON) res.bwd_tables = true;   // the polygon scan lives in that variant too
    if (!(kind_ok || forbes || grid) || o.coating == OLB_COAT_FRESNEL || tab.n_wl != 1)
      res.bwd_supported = false;
  }
  build_blob<double>(tab, pools, ps, features, polygons, res.blob_f64);
  build_blob<float>(tab, pools, ps, features, polygons, res.blob_f32);
  return res;
}

// ---- batched systems (SURVEY.md 8f-4): B perturbed copies of one template -----------------------------------
// `params`: n_systems x n_surfaces blocks of OLB_BP_COUNT doubles with ABSOLUTE values (include/olb.h).  Every
// system is prepared like a single table; the blobs must come out the same size (same structure) and are laid
// side by side; each header is stamped with the UNION of the feature bits (one kernel variant serves them all).
struct BatchPrep {
  std::vector<unsigned char> all64, all32;
  uint32_t features = 0, hints = 0;
  int32_t bytes_f64 = 0, bytes_f32 = 0;
  bool unsupported = false;
  std::string error;
};

static BatchPrep prepare_batch(const OlbTable& tmpl, const double* params, int n_systems) {
  BatchPrep out;
  if (tmpl.n_wl != 1) { out.error = "batched tables support one wavelength"; out.unsupported = true; return out; }
  const int S = tmpl.n_surfaces;
  for (int s = 0; s < S && tmpl.surfaces; ++s)
    if (tmpl.surfaces[s].interaction != OLB_INTERACT_REFRACT) {
      out.error = "batched tables with phase-profile or grating surfaces are not built"; out.unsupported = true; return out;
    }
  for (int s = 0; s < S && tmpl.surfaces; ++s)
    if (tmpl.surfaces[s].flags & OLB_SF_BSDF) {
      out.error = "batched tables with BSDF surfaces are not built"; out.unsupported = true; return out;
    }
  for (int s = 0; s < S && tmpl.surfaces; ++s)
    if (tmpl.surfaces[s].kind == OLB_GEOM_GRID_SAG) {
      out.error = "batched tables with grid-sag surfaces are not built"; out.unsupported = true; return out;
    }
  for (int s = 0; s < S && tmpl.surfaces; ++s)
    if (tmpl.surfaces[s].kind == OLB_GEOM_FORBES_Q2D) {
      out.error = "batched tables with Forbes Q-2D surfaces are not built"; out.unsupported = true; return out;
    }
  for (int s = 0; s < S && tmpl.surfaces; ++s)
    if (tmpl.surfaces[s].coating >= OLB_COAT_THIN_FILM && tmpl.surfaces[s].coating <= OLB_COAT_RETARDER) {
      out.error = "batched tables with thin-film, polarizer or retarder coatings are not built"; out.unsupported = true; return out;
    }
  std::vector<OlbSurface> surf(tmpl.surfaces, tmpl.surfaces + S);
  std::vector<double> pool(tmpl.pool, tmpl.pool + tmpl.pool_len);
  OlbTable t = tmpl;
  t.surfaces = surf.data();
  t.pool = pool.data();
  for (int b = 0; b < n_systems; ++b) {
    for (int s = 0; s < S; ++s) {
      const double* p = params + ((size_t)b * S + s) * OLB_BP_COUNT;
      OlbSurface& o = surf[s];
      const OlbSurface& o0 = tmpl.surfaces[s];
      if (o0.kind == OLB_GEOM_NOOP) continue;
      o.t[0] = p[OLB_BP_TX]; o.t[1] = p[OLB_BP_TY]; o.t[2] = p[OLB_BP_TZ];
      for (int q = 0; q < 9; ++q) o.R[q] = p[OLB_BP_R + q];
      if (o0.kind != OLB_GEOM_PLANE) {
        o.radius = p[OLB_BP_CURV] == 0 ? INFINITY : 1.0 / p[OLB_BP_CURV];
        if (o0.kind != OLB_GEOM_TOROIDAL) o.conic = p[OLB_BP_CONIC];
      }
      // media block (one wavelength): {n1, n2, k1, coating n1, coating n2}; without a Fresnel coating the last two
      // mirror n1 / n2 (table.py::pack)
      pool[o0.media_off + 0] = p[OLB_BP_N1];
      pool[o0.media_off + 1] = p[OLB_BP_N2];
      if (o0.coating != OLB_COAT_FRESNEL) {
        pool[o0.media_off + 3] = p[OLB_BP_N1];
        pool[o0.media_off + 4] = p[OLB_BP_N2];
      }
      if (o0.kind == OLB_GEOM_EVEN_ASPHERE)
        for (int j = 0; j < o0.n_coef && j < OLB_BP_MAX_COEF; ++j) pool[o0.coef_off + j] = p[OLB_BP_COEF + j];
    }
    PrepResult pr = prepare_table(t);
    if (!pr.error.empty()) { out.error = "system " + std::to_string(b) + ": " + pr.error; return out; }
    if (b == 0) {
      out.bytes_f64 = (int32_t)pr.blob_f64.size();
      out.bytes_f32 = (int32_t)pr.blob_f32.size();
    } else if ((int32_t)pr.blob_f64.size() != out.bytes_f64 || (int32_t)pr.blob_f32.size() != out.bytes_f32) {
      out.error = "batched systems must share one table structure";
      return out;
    }
    out.features |= pr.features;
    out.hints |= pr.hints;
    out.all64.insert(out.all64.end(), pr.blob_f64.begin(), pr.blob_f64.end());
    out.all32.insert(out.all32.end(), pr.blob_f32.begin(), pr.blob_f32.end());
  }
  for (int b = 0; b < n_systems; ++b) {
    reinterpret_cast<PrepHeader*>(out.all64.data() + (size_t)b * out.bytes_f64)->features = out.features;
    reinterpret_cast<PrepHeader*>(out.all32.data() + (size_t)b * out.bytes_f32)->features = out.features;
  }
  return out;
}

}  // namespace olb
#endif  // OLB_PREP_H_
