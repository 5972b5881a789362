// TEST INFRASTRUCTURE ONLY -- the CPU instantiation of the device arithmetic (hostcheck_grating.cpp, included whole,
// which includes hostcheck_phase.cpp and hostcheck.cpp) plus the kernel variant for tables with a thin-film, polarizer
// or retarder coating (FEAT_JONES): the general polarized kernel + FEAT_PHASE + FEAT_GRATING + FEAT_JONES, the
// instantiation the launcher picks for such tables (olb_trace.cu::launch_feat).  It also exports the per-ray Jones
// arithmetic of the thin-film stack on its own.  Built as its own library (_hostcheck_coating.so,
// oracle/hostcheck_coating.py); never linked into libolb.so.
#include "hostcheck_grating.cpp"

template <typename T>
static int run_coating(const OlbTable* tab, int first, int last, int64_t n, T** ray, T** rec, T** l0, T* pmat,
                       int* status, char* err, int err_len) {
  PrepResult pr = prepare_table(*tab);
  if (!pr.error.empty()) { snprintf(err, err_len, "%s", pr.error.c_str()); return OLB_ERR_TABLE; }
  if (!(pr.features & FEAT_JONES)) return run_grating<T>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len);
  const unsigned char* blob = sizeof(T) == 8 ? pr.blob_f64.data() : pr.blob_f32.data();
  if (!pmat) { snprintf(err, err_len, "table needs polarized rays (p)"); return OLB_ERR_INVALID_ARG; }
  constexpr uint32_t G = FEAT_ROT | FEAT_NEWTON | FEAT_EXTRA | FEAT_FREEFORM | FEAT_PHASE | FEAT_GRATING;
  walk<T, G | FEAT_POL | FEAT_JONES>(blob, first, last, n, ray, rec, l0, pmat, status);
  return OLB_OK;
}

// The thin-film Jones diagonal of surface `surf` of `tab` (which must carry a thin-film coating) for n rays at
// wavelength index widx[k] and angle of incidence aoi[k] (radians): out[k] = {Re r_s, Im r_s, Re t_s, Im t_s,
// Re r_p, Im r_p, Re t_p, Im t_p} in the reference's convention (thin_film/core.py:_tmm_coh; no sign flip of r_p).
template <typename T>
static int film_rt(const OlbTable* tab, int surf, int64_t n, const int* widx, const double* aoi, double* out,
                   char* err, int err_len) {
  PrepResult pr = prepare_table(*tab);
  if (!pr.error.empty()) { snprintf(err, err_len, "%s", pr.error.c_str()); return OLB_ERR_TABLE; }
  if (surf < 0 || surf >= tab->n_surfaces || tab->surfaces[surf].coating != OLB_COAT_THIN_FILM) {
    snprintf(err, err_len, "surface %d has no thin-film coating", surf); return OLB_ERR_INVALID_ARG;
  }
  const unsigned char* blob = sizeof(T) == 8 ? pr.blob_f64.data() : pr.blob_f32.data();
  const PrepHeader* H = reinterpret_cast<const PrepHeader*>(blob);
  const PrepSurface<T>* S = reinterpret_cast<const PrepSurface<T>*>(blob + sizeof(PrepHeader));
  const T* pool = reinterpret_cast<const T*>(S + H->n_surf);
  const T* hdr = pool + S[surf].media_off - CO_HDR;
  for (int64_t k = 0; k < n; ++k) {
    const T c = (T)std::cos(aoi[k]);
    Cx<T> rs, rp, ts, tp;
    thin_film_jones(hdr, widx[k], c * c, true, rs, rp);
    thin_film_jones(hdr, widx[k], c * c, false, ts, tp);
    double* o = out + 8 * k;
    o[0] = rs.re; o[1] = rs.im; o[2] = ts.re; o[3] = ts.im; o[4] = -(double)rp.re; o[5] = -(double)rp.im; o[6] = tp.re; o[7] = tp.im;
  }
  return OLB_OK;
}

extern "C" {
// same arguments as olbhc_trace_f64 / _f32; tables without these coatings take hostcheck_grating.cpp's dispatch
int olbhc_coating_trace_f64(const OlbTable* tab, int first, int last, int64_t n, double** ray, double** rec,
                            double** l0, double* pmat, int* status, char* err, int err_len) {
  return run_coating<double>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len);
}
int olbhc_coating_trace_f32(const OlbTable* tab, int first, int last, int64_t n, float** ray, float** rec,
                            float** l0, float* pmat, int* status, char* err, int err_len) {
  return run_coating<float>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len);
}
int olbhc_film_rt_f64(const OlbTable* tab, int surf, int64_t n, const int* widx, const double* aoi, double* out,
                      char* err, int err_len) {
  return film_rt<double>(tab, surf, n, widx, aoi, out, err, err_len);
}
int olbhc_film_rt_f32(const OlbTable* tab, int surf, int64_t n, const int* widx, const double* aoi, double* out,
                      char* err, int err_len) {
  return film_rt<float>(tab, surf, n, widx, aoi, out, err, err_len);
}
}
