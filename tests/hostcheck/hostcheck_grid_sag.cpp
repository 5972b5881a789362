// TEST INFRASTRUCTURE ONLY -- the CPU instantiation of the device arithmetic (hostcheck_coating.cpp, included whole,
// which includes the grating, phase and base host checks) plus the kernel variants for tables with a grid-sag surface
// (FEAT_GRID): the general kernel + FEAT_PHASE + FEAT_GRATING + FEAT_GRID and its polarized form with FEAT_JONES, the
// two instantiations the launcher picks for such tables (olb_trace.cu::launch_feat).  Built as its own library
// (_hostcheck_grid_sag.so, oracle/hostcheck_grid_sag.py); never linked into libolb.so.  The adjoint of grid tables is
// hostcheck.cpp's olbhc_backward_tables_*, whose surface_backward is the general (POLY) variant that covers them.
#include "hostcheck_coating.cpp"

template <typename T>
static int run_grid_sag(const OlbTable* tab, int first, int last, int64_t n, T** ray, T** rec, T** l0, T* pmat,
                        int* status, char* err, int err_len) {
  PrepResult pr = prepare_table(*tab);
  if (!pr.error.empty()) { snprintf(err, err_len, "%s", pr.error.c_str()); return OLB_ERR_TABLE; }
  if (!(pr.features & FEAT_GRID)) return run_coating<T>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len);
  const unsigned char* blob = sizeof(T) == 8 ? pr.blob_f64.data() : pr.blob_f32.data();
  if ((pr.features & FEAT_POL) && !pmat) { snprintf(err, err_len, "table needs polarized rays (p)"); return OLB_ERR_INVALID_ARG; }
  constexpr uint32_t G = FEAT_ROT | FEAT_NEWTON | FEAT_EXTRA | FEAT_FREEFORM | FEAT_PHASE | FEAT_GRATING | FEAT_GRID;
  if (pmat) walk<T, G | FEAT_POL | FEAT_JONES>(blob, first, last, n, ray, rec, l0, pmat, status);
  else walk<T, G>(blob, first, last, n, ray, rec, l0, nullptr, status);
  return OLB_OK;
}

extern "C" {
// same arguments as olbhc_trace_f64 / _f32; tables without a grid-sag surface take hostcheck_coating.cpp's dispatch
int olbhc_grid_sag_trace_f64(const OlbTable* tab, int first, int last, int64_t n, double** ray, double** rec,
                             double** l0, double* pmat, int* status, char* err, int err_len) {
  return run_grid_sag<double>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len);
}
int olbhc_grid_sag_trace_f32(const OlbTable* tab, int first, int last, int64_t n, float** ray, float** rec,
                             float** l0, float* pmat, int* status, char* err, int err_len) {
  return run_grid_sag<float>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len);
}
}
