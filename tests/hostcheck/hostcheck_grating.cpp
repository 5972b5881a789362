// TEST INFRASTRUCTURE ONLY -- the CPU instantiation of the device arithmetic (hostcheck_phase.cpp, included whole,
// which includes hostcheck.cpp) plus the kernel variants for tables with a ruled grating (FEAT_GRATING): the general
// kernel + FEAT_PHASE + FEAT_GRATING and its polarized form, the two instantiations the launcher picks for such tables
// (olb_trace.cu::launch_feat).  Built as its own library (_hostcheck_grating.so, oracle/hostcheck_grating.py); never
// linked into libolb.so.
#include "hostcheck_phase.cpp"

template <typename T>
static int run_grating(const OlbTable* tab, int first, int last, int64_t n, T** ray, T** rec, T** l0, T* pmat,
                       int* status, char* err, int err_len) {
  PrepResult pr = prepare_table(*tab);
  if (!pr.error.empty()) { snprintf(err, err_len, "%s", pr.error.c_str()); return OLB_ERR_TABLE; }
  if (!(pr.features & FEAT_GRATING)) return run_phase<T>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len);
  const unsigned char* blob = sizeof(T) == 8 ? pr.blob_f64.data() : pr.blob_f32.data();
  if ((pr.features & FEAT_POL) && !pmat) { snprintf(err, err_len, "table needs polarized rays (p)"); return OLB_ERR_INVALID_ARG; }
  constexpr uint32_t G = FEAT_ROT | FEAT_NEWTON | FEAT_EXTRA | FEAT_FREEFORM | FEAT_PHASE | FEAT_GRATING;
  if (pmat) walk<T, G | FEAT_POL>(blob, first, last, n, ray, rec, l0, pmat, status);
  else walk<T, G>(blob, first, last, n, ray, rec, l0, nullptr, status);
  return OLB_OK;
}

extern "C" {
// same arguments as olbhc_trace_f64 / _f32; tables without a grating take hostcheck_phase.cpp's dispatch
int olbhc_grating_trace_f64(const OlbTable* tab, int first, int last, int64_t n, double** ray, double** rec,
                            double** l0, double* pmat, int* status, char* err, int err_len) {
  return run_grating<double>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len);
}
int olbhc_grating_trace_f32(const OlbTable* tab, int first, int last, int64_t n, float** ray, float** rec,
                            float** l0, float* pmat, int* status, char* err, int err_len) {
  return run_grating<float>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len);
}
}
