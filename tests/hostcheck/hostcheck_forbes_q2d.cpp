// TEST INFRASTRUCTURE ONLY -- the CPU instantiation of the device arithmetic (hostcheck_coating.cpp, included whole,
// which includes the grating, phase and base host checks) plus the two kernel variants of tables with a Forbes Q-2D
// surface (FEAT_Q2D): the general kernel + FEAT_Q2D and the general polarized kernel + FEAT_Q2D, the instantiations the
// launcher picks for such tables (olb_trace.cu::launch_feat).  Built as its own library (_hostcheck_forbes_q2d.so,
// oracle/hostcheck_forbes_q2d.py); never linked into libolb.so.
#include "hostcheck_coating.cpp"

template <typename T>
static int run_forbes_q2d(const OlbTable* tab, int first, int last, int64_t n, T** ray, T** rec, T** l0, T* pmat,
                          int* status, char* err, int err_len) {
  PrepResult pr = prepare_table(*tab);
  if (!pr.error.empty()) { snprintf(err, err_len, "%s", pr.error.c_str()); return OLB_ERR_TABLE; }
  if (!(pr.features & FEAT_Q2D)) return run_coating<T>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len);
  constexpr uint32_t EXCLUDED = FEAT_PHASE | FEAT_GRATING | FEAT_GRID | FEAT_POLYGON | FEAT_BSDF | FEAT_JONES;
  if (pr.features & EXCLUDED) { snprintf(err, err_len, "Forbes Q-2D beside an excluded feature"); return OLB_ERR_UNSUPPORTED; }
  const unsigned char* blob = sizeof(T) == 8 ? pr.blob_f64.data() : pr.blob_f32.data();
  if ((pr.features & FEAT_POL) && !pmat) { snprintf(err, err_len, "table needs polarized rays (p)"); return OLB_ERR_INVALID_ARG; }
  constexpr uint32_t G = FEAT_ROT | FEAT_NEWTON | FEAT_EXTRA | FEAT_FREEFORM | FEAT_Q2D;
  if (pmat) walk<T, G | FEAT_POL>(blob, first, last, n, ray, rec, l0, pmat, status);
  else walk<T, G>(blob, first, last, n, ray, rec, l0, nullptr, status);
  return OLB_OK;
}

// Sag and slopes of surface `surf` (a Q-2D surface) at n local points, as the kernel evaluates them.
template <typename T>
static int forbes_q2d_eval(const OlbTable* tab, int surf, int64_t n, const double* x, const double* y, double* sag,
                           double* fx, double* fy, char* err, int err_len) {
  PrepResult pr = prepare_table(*tab);
  if (!pr.error.empty()) { snprintf(err, err_len, "%s", pr.error.c_str()); return OLB_ERR_TABLE; }
  if (surf < 0 || surf >= tab->n_surfaces || tab->surfaces[surf].kind != OLB_GEOM_FORBES_Q2D) {
    snprintf(err, err_len, "surface %d is not a Forbes Q-2D surface", surf); return OLB_ERR_INVALID_ARG;
  }
  const unsigned char* blob = sizeof(T) == 8 ? pr.blob_f64.data() : pr.blob_f32.data();
  const PrepHeader* H = reinterpret_cast<const PrepHeader*>(blob);
  const PrepSurface<T>* S = reinterpret_cast<const PrepSurface<T>*>(blob + sizeof(PrepHeader));
  const T* pool = reinterpret_cast<const T*>(S + H->n_surf);
  for (int64_t k = 0; k < n; ++k) {
    T gx, gy;
    sag[k] = q2d_sag<T>((T)x[k], (T)y[k], S[surf], pool);
    q2d_slopes<T>((T)x[k], (T)y[k], S[surf], pool, gx, gy);
    fx[k] = gx; fy[k] = gy;
  }
  return OLB_OK;
}

extern "C" {
// same arguments as olbhc_trace_f64 / _f32; tables without a Q-2D surface take hostcheck_coating.cpp's dispatch
int olbhc_forbes_q2d_trace_f64(const OlbTable* tab, int first, int last, int64_t n, double** ray, double** rec,
                               double** l0, double* pmat, int* status, char* err, int err_len) {
  return run_forbes_q2d<double>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len);
}
int olbhc_forbes_q2d_trace_f32(const OlbTable* tab, int first, int last, int64_t n, float** ray, float** rec,
                               float** l0, float* pmat, int* status, char* err, int err_len) {
  return run_forbes_q2d<float>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len);
}
int olbhc_forbes_q2d_eval_f64(const OlbTable* tab, int surf, int64_t n, const double* x, const double* y, double* sag,
                              double* fx, double* fy, char* err, int err_len) {
  return forbes_q2d_eval<double>(tab, surf, n, x, y, sag, fx, fy, err, err_len);
}
int olbhc_forbes_q2d_eval_f32(const OlbTable* tab, int surf, int64_t n, const double* x, const double* y, double* sag,
                              double* fx, double* fy, char* err, int err_len) {
  return forbes_q2d_eval<float>(tab, surf, n, x, y, sag, fx, fy, err, err_len);
}
}
