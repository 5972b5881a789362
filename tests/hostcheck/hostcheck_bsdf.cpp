// TEST INFRASTRUCTURE ONLY -- the CPU instantiation of the device arithmetic (hostcheck_polygon.cpp, included whole,
// which includes the grid-sag, coating, grating, phase and base host checks) plus the kernel variant for tables with a
// BSDF surface (FEAT_BSDF): the polygon superset + the scatter step of olb_bsdf.cuh, the instantiation the launcher
// picks for such tables (olb_trace.cu::launch_feat).  It also exports the draw function, so that tests can drive the
// reference's own scatter with the kernel's random numbers.  Built as its own library (_hostcheck_bsdf.so,
// oracle/hostcheck_bsdf.py); never linked into libolb.so.
#include "hostcheck_polygon.cpp"
#include "../../optiland_b200/csrc/olb_bsdf.cuh"

// hostcheck.cpp's walk, with the ray index (ray0 + k) and the call's stream that key the scatter draws
template <typename T, uint32_t FEAT>
static void walk_bsdf(const unsigned char* blob, int first, int last, int64_t n, T** ray, T** rec, T** l0, int64_t ray0,
                      uint32_t stream, int* status_out) {
  const PrepHeader* H = reinterpret_cast<const PrepHeader*>(blob);
  const PrepSurface<T>* surf = reinterpret_cast<const PrepSurface<T>*>(blob + sizeof(PrepHeader));
  const T* pool = reinterpret_cast<const T*>(surf + H->n_surf);
  const T* wl = pool + H->pad[0];
  int status = 0;
  for (int64_t k = 0; k < n; ++k) {
    Ray<T> r{};
    r.x = ray[0][k]; r.y = ray[1][k]; r.z = ray[2][k]; r.L = ray[3][k]; r.M = ray[4][k]; r.N = ray[5][k];
    r.i = ray[6][k]; r.opd = ray[8][k]; r.opd_lo = 0; r.widx = 0;
    r.id = (uint64_t)(ray0 + k); r.stream = stream;
    if (H->n_wl > 1) {
      int idx = -1;
      for (int j = 0; j < H->n_wl; ++j)
        if (ray[7][k] == wl[j]) idx = j;
      r.widx = idx;
    }
    bool have_frame = false;
    T g[6] = {r.x, r.y, r.z, r.L, r.M, r.N};
    for (int s = first; s < last; ++s) {
      const PrepSurface<T>& S = surf[s];
      const bool noop = S.kind == OLB_GEOM_NOOP;
      if (!noop) { surface_step<T, FEAT>(r, S, pool, !have_frame, status, nullptr, 1); have_frame = true; }
      const bool record = rec != nullptr && !(S.flags & OLB_SF_NORECORD);
      if ((record || s == last - 1) && !noop) to_global<T, FEAT>(r, S, g[0], g[1], g[2], g[3], g[4], g[5]);
      if (record) {
        const int64_t off = (int64_t)(s - first) * n + k;
        for (int q = 0; q < 6; ++q) rec[q][off] = g[q];
        rec[6][off] = r.i;
        rec[7][off] = opd_value(r);
      }
    }
    for (int q = 0; q < 6; ++q) ray[q][k] = g[q];
    ray[6][k] = r.i;
    ray[8][k] = opd_value(r);
    if (l0) { l0[0][k] = r.L0; l0[1][k] = r.M0; l0[2][k] = r.N0; }
  }
  *status_out |= status;
}

template <typename T>
static int run_bsdf(const OlbTable* tab, int first, int last, int64_t n, T** ray, T** rec, T** l0, T* pmat,
                    int* status, char* err, int err_len, int64_t ray0, uint32_t stream) {
  PrepResult pr = prepare_table(*tab);
  if (!pr.error.empty()) { snprintf(err, err_len, "%s", pr.error.c_str()); return OLB_ERR_TABLE; }
  if (!(pr.features & FEAT_BSDF)) return run_polygon<T>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len);
  if ((pr.features & FEAT_POL) || pmat) {
    snprintf(err, err_len, "polarized trace of a table with a BSDF surface is not built");
    return OLB_ERR_UNSUPPORTED;
  }
  const unsigned char* blob = sizeof(T) == 8 ? pr.blob_f64.data() : pr.blob_f32.data();
  constexpr uint32_t G = FEAT_ROT | FEAT_NEWTON | FEAT_EXTRA | FEAT_FREEFORM | FEAT_PHASE | FEAT_GRATING | FEAT_GRID |
                         FEAT_POLYGON | FEAT_BSDF;
  walk_bsdf<T, G>(blob, first, last, n, ray, rec, l0, ray0, stream, status);
  return OLB_OK;
}

extern "C" {
// olbhc_trace_f64 / _f32's arguments, then the index of the first ray and the call's rng_stream; tables without a BSDF
// take hostcheck_polygon.cpp's dispatch
int olbhc_bsdf_trace_f64(const OlbTable* tab, int first, int last, int64_t n, double** ray, double** rec, double** l0,
                         double* pmat, int* status, char* err, int err_len, int64_t ray0, uint32_t stream) {
  return run_bsdf<double>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len, ray0, stream);
}
int olbhc_bsdf_trace_f32(const OlbTable* tab, int first, int last, int64_t n, float** ray, float** rec, float** l0,
                         float* pmat, int* status, char* err, int err_len, int64_t ray0, uint32_t stream) {
  return run_bsdf<float>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len, ray0, stream);
}
// Draws attempt0 .. attempt0 + count - 1 of ray `ray`: xy[2 j], xy[2 j + 1] = (x, y) of draw attempt0 + j, computed in
// fp64 (which = 0) or fp32 (which = 1) exactly as the kernel draws them.  `seed` is the surface's 64-bit key.
int olbhc_bsdf_draws(uint64_t seed, uint32_t stream, uint64_t ray, uint32_t attempt0, int count, int kind, double sigma,
                     int which, double* xy) {
  for (int j = 0; j < count; ++j) {
    if (which == 0) {
      double x, y;
      bsdf_draw<double>(seed, ray, stream, attempt0 + (uint32_t)j, kind, sigma, x, y);
      xy[2 * j] = x; xy[2 * j + 1] = y;
    } else {
      float x, y;
      bsdf_draw<float>(seed, ray, stream, attempt0 + (uint32_t)j, kind, (float)sigma, x, y);
      xy[2 * j] = x; xy[2 * j + 1] = y;
    }
  }
  return 0;
}
// One Philox4x32-10 block, for the known-answer test of the host instantiation
void olbhc_philox(const uint32_t* ctr, const uint32_t* key, uint32_t* out) {
  uint4 c; c.x = ctr[0]; c.y = ctr[1]; c.z = ctr[2]; c.w = ctr[3];
  uint2 k; k.x = key[0]; k.y = key[1];
  const uint4 o = curand_Philox4x32_10(c, k);
  out[0] = o.x; out[1] = o.y; out[2] = o.z; out[3] = o.w;
}
}
