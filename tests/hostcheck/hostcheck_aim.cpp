// TEST INFRASTRUCTURE ONLY -- the CPU instantiation of the ray-aiming solve (olb_aim.cuh) with the three kernel
// variants olb_trace.cu::aim_impl picks (closed form, general, phase / grating / grid-sag / polygon superset), on top
// of hostcheck_polygon.cpp (included whole).  Built as its own library (_hostcheck_aim.so, oracle/hostcheck_aim.py);
// never linked into libolb.so.
#include "hostcheck_polygon.cpp"
#include "../../optiland_b200/csrc/olb_aim.cuh"

template <typename T>
static int aim_widx_of(const unsigned char* blob, T w) {
  const PrepHeader* H = reinterpret_cast<const PrepHeader*>(blob);
  const PrepSurface<T>* surf = reinterpret_cast<const PrepSurface<T>*>(blob + sizeof(PrepHeader));
  const T* wl = reinterpret_cast<const T*>(surf + H->n_surf) + H->pad[0];
  return H->n_wl > 1 ? aim_widx<T>(wl, H->n_wl, w) : 0;
}

template <typename T, uint32_t FEAT>
static void aim_walk(const unsigned char* blob, int first, int last, int64_t n, T** g, const T* px, const T* py,
                     double r_stop, double J, double tol, int max_iter, int infinite, int* status_out, int* ray_status) {
  const PrepHeader* H = reinterpret_cast<const PrepHeader*>(blob);
  const PrepSurface<T>* surf = reinterpret_cast<const PrepSurface<T>*>(blob + sizeof(PrepHeader));
  const T* pool = reinterpret_cast<const T*>(surf + H->n_surf);
  const T rs = (T)r_stop, Jf = (T)J, tol_sq = (T)(tol * tol);
  int status = 0;
  for (int64_t k = 0; k < n; ++k) {
    T x = g[0][k], y = g[1][k], L = g[3][k], M = g[4][k];
    const int s = aim_ray<T, FEAT>(surf, pool, first, last, x, y, g[2][k], L, M, g[5][k], aim_widx_of<T>(blob, g[6][k]),
                                   o_mul_nc(px[k], rs), o_mul_nc(py[k], rs), Jf, tol_sq, max_iter, infinite != 0);
    if (ray_status) ray_status[k] = s;
    status |= s;
    if (infinite) { g[0][k] = x; g[1][k] = y; }
    else { g[3][k] = L; g[4][k] = M; }
  }
  *status_out |= status;
}

// The stop-local residual (x_s - Px r_stop, y_s - Py r_stop) of each launch state, as aim_ray forms it before a step.
template <typename T, uint32_t FEAT>
static void aim_residual_walk(const unsigned char* blob, int first, int last, int64_t n, T** g, const T* px,
                              const T* py, double r_stop, T* ex, T* ey, int* status_out) {
  const PrepHeader* H = reinterpret_cast<const PrepHeader*>(blob);
  const PrepSurface<T>* surf = reinterpret_cast<const PrepSurface<T>*>(blob + sizeof(PrepHeader));
  const T* pool = reinterpret_cast<const T*>(surf + H->n_surf);
  const T rs = (T)r_stop;
  int status = 0;
  for (int64_t k = 0; k < n; ++k) {
    T lx, ly;
    aim_trace<T, FEAT>(surf, pool, first, last, g[0][k], g[1][k], g[2][k], g[3][k], g[4][k], g[5][k],
                       aim_widx_of<T>(blob, g[6][k]), lx, ly, status);
    ex[k] = lx - o_mul_nc(px[k], rs);
    ey[k] = ly - o_mul_nc(py[k], rs);
  }
  *status_out |= status;
}

// residual == 0: solve (aim_walk); residual == 1: only the residuals of the given launch states (aim_residual_walk).
template <typename T>
static int run_aim(const OlbTable* tab, int first, int last, int64_t n, T** g, const T* px, const T* py, double r_stop,
                   double J, double tol, int max_iter, int infinite, int* status, int* variant, int* ray_status, T* ex,
                   T* ey, char* err, int err_len) {
  PrepResult pr = prepare_table(*tab);
  if (!pr.error.empty()) { snprintf(err, err_len, "%s", pr.error.c_str()); return OLB_ERR_TABLE; }
  if (first < 0 || last > tab->n_surfaces || first >= last) { snprintf(err, err_len, "bad surface range"); return OLB_ERR_INVALID_ARG; }
  const int v = aim_variant(pr.features);
  *variant = v;
  if (v < 0) { snprintf(err, err_len, "ray aiming through a BSDF surface or a polarizing coating is not built"); return OLB_ERR_UNSUPPORTED; }
  const unsigned char* blob = sizeof(T) == 8 ? pr.blob_f64.data() : pr.blob_f32.data();
  if (ex) {
    if (v == AIM_CLOSED_FORM) aim_residual_walk<T, FEAT_ROT>(blob, first, last, n, g, px, py, r_stop, ex, ey, status);
    else if (v == AIM_GENERAL) aim_residual_walk<T, AIM_FEAT_GENERAL>(blob, first, last, n, g, px, py, r_stop, ex, ey, status);
    else aim_residual_walk<T, AIM_FEAT_SUPERSET>(blob, first, last, n, g, px, py, r_stop, ex, ey, status);
    return OLB_OK;
  }
  if (v == AIM_CLOSED_FORM) aim_walk<T, FEAT_ROT>(blob, first, last, n, g, px, py, r_stop, J, tol, max_iter, infinite, status, ray_status);
  else if (v == AIM_GENERAL) aim_walk<T, AIM_FEAT_GENERAL>(blob, first, last, n, g, px, py, r_stop, J, tol, max_iter, infinite, status, ray_status);
  else aim_walk<T, AIM_FEAT_SUPERSET>(blob, first, last, n, g, px, py, r_stop, J, tol, max_iter, infinite, status, ray_status);
  return OLB_OK;
}

extern "C" {
// g: 7 arrays x, y, z, L, M, N, w of n values (w read only for tables with several wavelengths); the solution is written
// into x, y (infinite) or L, M.  *variant receives the kernel variant (AIM_*; -1 not built).  ray_status (optional, n
// int32): each ray's own OLB_ST_* bits, whose OR is *status.
int olbhc_aim_f64(const OlbTable* tab, int first, int last, int64_t n, double** g, const double* px, const double* py,
                  double r_stop, double J, double tol, int max_iter, int infinite, int* status, int* variant,
                  int* ray_status, char* err, int err_len) {
  return run_aim<double>(tab, first, last, n, g, px, py, r_stop, J, tol, max_iter, infinite, status, variant, ray_status,
                         nullptr, nullptr, err, err_len);
}
int olbhc_aim_f32(const OlbTable* tab, int first, int last, int64_t n, float** g, const float* px, const float* py,
                  double r_stop, double J, double tol, int max_iter, int infinite, int* status, int* variant,
                  int* ray_status, char* err, int err_len) {
  return run_aim<float>(tab, first, last, n, g, px, py, r_stop, J, tol, max_iter, infinite, status, variant, ray_status,
                        nullptr, nullptr, err, err_len);
}
// The residual on the stop of each launch state in g (no step): ex, ey receive n values each.
int olbhc_aim_residual_f64(const OlbTable* tab, int first, int last, int64_t n, double** g, const double* px,
                           const double* py, double r_stop, double* ex, double* ey, int* status, char* err, int err_len) {
  int variant = -1;
  return run_aim<double>(tab, first, last, n, g, px, py, r_stop, 0.0, 0.0, 0, 1, status, &variant, nullptr, ex, ey, err,
                         err_len);
}
int olbhc_aim_residual_f32(const OlbTable* tab, int first, int last, int64_t n, float** g, const float* px,
                           const float* py, double r_stop, float* ex, float* ey, int* status, char* err, int err_len) {
  int variant = -1;
  return run_aim<float>(tab, first, last, n, g, px, py, r_stop, 0.0, 0.0, 0, 1, status, &variant, nullptr, ex, ey, err,
                        err_len);
}
}
