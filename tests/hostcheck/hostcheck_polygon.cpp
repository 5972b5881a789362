// TEST INFRASTRUCTURE ONLY -- the CPU instantiation of the device arithmetic (hostcheck_grid_sag.cpp, included whole,
// which includes the coating, grating, phase and base host checks) plus the kernel variants for tables with a polygon
// in an aperture program (FEAT_POLYGON): the grid-sag superset + FEAT_POLYGON and its polarized form, the two
// instantiations the launcher picks for such tables (olb_trace.cu::launch_feat).  Built as its own library
// (_hostcheck_polygon.so, oracle/hostcheck_polygon.py); never linked into libolb.so.  The adjoint of polygon tables is
// hostcheck.cpp's olbhc_backward_tables_*, whose surface_backward is the general (POLY) variant that holds the scan.
#include "hostcheck_grid_sag.cpp"

template <typename T>
static int run_polygon(const OlbTable* tab, int first, int last, int64_t n, T** ray, T** rec, T** l0, T* pmat,
                       int* status, char* err, int err_len) {
  PrepResult pr = prepare_table(*tab);
  if (!pr.error.empty()) { snprintf(err, err_len, "%s", pr.error.c_str()); return OLB_ERR_TABLE; }
  if (!(pr.features & FEAT_POLYGON)) return run_grid_sag<T>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len);
  const unsigned char* blob = sizeof(T) == 8 ? pr.blob_f64.data() : pr.blob_f32.data();
  if ((pr.features & FEAT_POL) && !pmat) { snprintf(err, err_len, "table needs polarized rays (p)"); return OLB_ERR_INVALID_ARG; }
  constexpr uint32_t G = FEAT_ROT | FEAT_NEWTON | FEAT_EXTRA | FEAT_FREEFORM | FEAT_PHASE | FEAT_GRATING | FEAT_GRID | FEAT_POLYGON;
  if (pmat) walk<T, G | FEAT_POL | FEAT_JONES>(blob, first, last, n, ray, rec, l0, pmat, status);
  else walk<T, G>(blob, first, last, n, ray, rec, l0, nullptr, status);
  return OLB_OK;
}

extern "C" {
// same arguments as olbhc_trace_f64 / _f32; tables without a polygon take hostcheck_grid_sag.cpp's dispatch
int olbhc_polygon_trace_f64(const OlbTable* tab, int first, int last, int64_t n, double** ray, double** rec,
                            double** l0, double* pmat, int* status, char* err, int err_len) {
  return run_polygon<double>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len);
}
int olbhc_polygon_trace_f32(const OlbTable* tab, int first, int last, int64_t n, float** ray, float** rec,
                            float** l0, float* pmat, int* status, char* err, int err_len) {
  return run_polygon<float>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len);
}
// the prepared polygon of the table's surface `surface` (its first POLYGON instruction) in precision `which`
// (0: fp64, 1: fp32), as doubles: out = {buckets, ymin, ymax, records}, then `cap` values of the edge block
int olbhc_polygon_block(const OlbTable* tab, int surface, int which, double* out, int cap, char* err, int err_len) {
  PrepResult pr = prepare_table(*tab);
  if (!pr.error.empty()) { snprintf(err, err_len, "%s", pr.error.c_str()); return -1; }
  auto dump = [&](auto zero, const std::vector<unsigned char>& blob) -> int {
    using T = decltype(zero);
    const PrepHeader* H = reinterpret_cast<const PrepHeader*>(blob.data());
    const PrepSurface<T>* surf = reinterpret_cast<const PrepSurface<T>*>(blob.data() + sizeof(PrepHeader));
    const T* pool = reinterpret_cast<const T*>(surf + H->n_surf);
    const T* prog = pool + surf[surface].aper_off;
    int i = 0;
    while (i < surf[surface].aper_len && (int)prog[i] != OLB_AP_POLYGON) i += 1 + aperture_operands((int)prog[i]);
    if (i >= surf[surface].aper_len) return -1;
    const T* pg = prog + i;
    const int nb = (int)pg[PG_NB];
    const T* start = pg + (int)pg[PG_OFF];
    const int records = (int)start[nb];
    out[0] = nb; out[1] = (double)pg[PG_YMIN]; out[2] = (double)pg[PG_YMAX]; out[3] = records;
    const int len = ((nb + 1 + 3) & ~3) + PG_REC * records;
    for (int k = 0; k < len && k + 4 < cap; ++k) out[4 + k] = (double)start[k];
    return len;
  };
  return which == 0 ? dump(0.0, pr.blob_f64) : dump(0.0f, pr.blob_f32);
}
}
