// TEST INFRASTRUCTURE ONLY -- the CPU instantiation of the ray-aiming solve (olb_aim.cuh) with the three kernel
// variants olb_trace.cu::aim_impl picks (closed form, general, phase / grating / grid-sag / polygon superset), on top
// of hostcheck_polygon.cpp (included whole).  Built as its own library (_hostcheck_aim.so, oracle/hostcheck_aim.py);
// never linked into libolb.so.
#include "hostcheck_polygon.cpp"
#include "../../optiland_b200/csrc/olb_aim.cuh"

template <typename T, uint32_t FEAT>
static void aim_walk(const unsigned char* blob, int first, int last, int64_t n, T** g, const T* px, const T* py,
                     double r_stop, double J, double tol, int max_iter, int infinite, int* status_out) {
  const PrepHeader* H = reinterpret_cast<const PrepHeader*>(blob);
  const PrepSurface<T>* surf = reinterpret_cast<const PrepSurface<T>*>(blob + sizeof(PrepHeader));
  const T* pool = reinterpret_cast<const T*>(surf + H->n_surf);
  const T* wl = pool + H->pad[0];
  const T rs = (T)r_stop, Jf = (T)J, tol_sq = (T)(tol * tol);
  int status = 0;
  for (int64_t k = 0; k < n; ++k) {
    T x = g[0][k], y = g[1][k], L = g[3][k], M = g[4][k];
    const int widx = H->n_wl > 1 ? aim_widx<T>(wl, H->n_wl, g[6][k]) : 0;
    status |= aim_ray<T, FEAT>(surf, pool, first, last, x, y, g[2][k], L, M, g[5][k], widx, o_mul_nc(px[k], rs),
                               o_mul_nc(py[k], rs), Jf, tol_sq, max_iter, infinite != 0);
    if (infinite) { g[0][k] = x; g[1][k] = y; }
    else { g[3][k] = L; g[4][k] = M; }
  }
  *status_out |= status;
}

template <typename T>
static int run_aim(const OlbTable* tab, int first, int last, int64_t n, T** g, const T* px, const T* py, double r_stop,
                   double J, double tol, int max_iter, int infinite, int* status, int* variant, char* err, int err_len) {
  PrepResult pr = prepare_table(*tab);
  if (!pr.error.empty()) { snprintf(err, err_len, "%s", pr.error.c_str()); return OLB_ERR_TABLE; }
  if (first < 0 || last > tab->n_surfaces || first >= last) { snprintf(err, err_len, "bad surface range"); return OLB_ERR_INVALID_ARG; }
  const int v = aim_variant(pr.features);
  *variant = v;
  if (v < 0) { snprintf(err, err_len, "ray aiming through a BSDF surface or a polarizing coating is not built"); return OLB_ERR_UNSUPPORTED; }
  const unsigned char* blob = sizeof(T) == 8 ? pr.blob_f64.data() : pr.blob_f32.data();
  if (v == AIM_CLOSED_FORM) aim_walk<T, FEAT_ROT>(blob, first, last, n, g, px, py, r_stop, J, tol, max_iter, infinite, status);
  else if (v == AIM_GENERAL) aim_walk<T, AIM_FEAT_GENERAL>(blob, first, last, n, g, px, py, r_stop, J, tol, max_iter, infinite, status);
  else aim_walk<T, AIM_FEAT_SUPERSET>(blob, first, last, n, g, px, py, r_stop, J, tol, max_iter, infinite, status);
  return OLB_OK;
}

extern "C" {
// g: 7 arrays x, y, z, L, M, N, w of n values (w read only for tables with several wavelengths); the solution is written
// into x, y (infinite) or L, M.  *variant receives the kernel variant (AIM_*; -1 not built).
int olbhc_aim_f64(const OlbTable* tab, int first, int last, int64_t n, double** g, const double* px, const double* py,
                  double r_stop, double J, double tol, int max_iter, int infinite, int* status, int* variant, char* err,
                  int err_len) {
  return run_aim<double>(tab, first, last, n, g, px, py, r_stop, J, tol, max_iter, infinite, status, variant, err, err_len);
}
int olbhc_aim_f32(const OlbTable* tab, int first, int last, int64_t n, float** g, const float* px, const float* py,
                  double r_stop, double J, double tol, int max_iter, int infinite, int* status, int* variant, char* err,
                  int err_len) {
  return run_aim<float>(tab, first, last, n, g, px, py, r_stop, J, tol, max_iter, infinite, status, variant, err, err_len);
}
}
