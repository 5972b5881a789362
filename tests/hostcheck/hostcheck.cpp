// TEST INFRASTRUCTURE ONLY -- CPU instantiation of the device arithmetic.
//
// olb_math.cuh (surface_step / to_global) and olb_prep.h (table preparation) are the
// exact sources libolb.so compiles for sm_90a; here they are compiled by g++ so the
// GPU-less build container can check the kernel arithmetic against the oracle
// (tests/test_hostcheck.py).  This object is never linked into libolb.so and the
// product package never loads it: it is not a CPU fallback.
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "../../optiland_b200/csrc/olb_math.cuh"
#include "../../optiland_b200/csrc/olb_fftpsf.cuh"

using namespace olb;

template <typename T, uint32_t FEAT>
static void walk(const unsigned char* blob, int first, int last, int64_t n, T** ray /*x y z L M N i w opd*/,
                 T** rec /*8 arrays rows*n or null*/, T** l0 /*3 or null*/, T* pmat /*[n][18] or null*/,
                 int* status_out) {
  const PrepHeader* H = reinterpret_cast<const PrepHeader*>(blob);
  const PrepSurface<T>* surf = reinterpret_cast<const PrepSurface<T>*>(blob + sizeof(PrepHeader));
  const T* pool = reinterpret_cast<const T*>(surf + H->n_surf);
  const T* wl = pool + H->pad[0];
  int status = 0;
  for (int64_t k = 0; k < n; ++k) {
    Ray<T> r{};
    r.x = ray[0][k]; r.y = ray[1][k]; r.z = ray[2][k]; r.L = ray[3][k]; r.M = ray[4][k]; r.N = ray[5][k];
    r.i = ray[6][k]; r.opd = ray[8][k]; r.opd_lo = 0; r.widx = 0;
    if (H->n_wl > 1) {
      int idx = -1;
      for (int j = 0; j < H->n_wl; ++j)
        if (ray[7][k] == wl[j]) idx = j;
      r.widx = idx;
    }
    if ((FEAT & FEAT_POL) && pmat)
      for (int q = 0; q < 18; ++q) r.P[q] = pmat[k * 18 + q];
    bool have_frame = false;
    T g[6] = {r.x, r.y, r.z, r.L, r.M, r.N};
    for (int s = first; s < last; ++s) {
      const PrepSurface<T>& S = surf[s];
      const bool noop = S.kind == OLB_GEOM_NOOP;
      if (!noop) { surface_step<T, FEAT>(r, S, pool, !have_frame, status, r.P, 1); have_frame = true; }
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
    if ((FEAT & FEAT_POL) && pmat)
      for (int q = 0; q < 18; ++q) pmat[k * 18 + q] = r.P[q];
  }
  *status_out |= status;
}

template <typename T>
static int run(const OlbTable* tab, int first, int last, int64_t n, T** ray, T** rec, T** l0, T* pmat,
               int* status, char* err, int err_len) {
  PrepResult pr = prepare_table(*tab);
  if (!pr.error.empty()) { snprintf(err, err_len, "%s", pr.error.c_str()); return OLB_ERR_TABLE; }
  const unsigned char* blob = sizeof(T) == 8 ? pr.blob_f64.data() : pr.blob_f32.data();
  if ((pr.features & FEAT_POL) && !pmat) { snprintf(err, err_len, "table needs polarized rays (p)"); return OLB_ERR_INVALID_ARG; }
  if (pmat) {
    walk<T, FEAT_ROT | FEAT_NEWTON | FEAT_EXTRA | FEAT_FREEFORM | FEAT_POL>(blob, first, last, n, ray, rec, l0, pmat, status);
    return OLB_OK;
  }
  // exercise the same instantiations the launcher picks from
  uint32_t f = pr.features | (l0 ? FEAT_EXTRA : 0u);
  if (f == 0) walk<T, 0u>(blob, first, last, n, ray, rec, l0, nullptr, status);
  else if (f == FEAT_ROT) walk<T, FEAT_ROT>(blob, first, last, n, ray, rec, l0, nullptr, status);
  else if (f == FEAT_NEWTON) walk<T, FEAT_NEWTON>(blob, first, last, n, ray, rec, l0, nullptr, status);
  else if (f == (FEAT_NEWTON | FEAT_FREEFORM)) walk<T, FEAT_NEWTON | FEAT_FREEFORM>(blob, first, last, n, ray, rec, l0, nullptr, status);
  else walk<T, FEAT_ROT | FEAT_NEWTON | FEAT_EXTRA | FEAT_FREEFORM>(blob, first, last, n, ray, rec, l0, nullptr, status);
  return OLB_OK;
}

// Reverse sweep over surfaces for every ray: the loop the backward kernel runs per thread.
template <typename T>
static int run_backward(const OlbTable* tab, int first, int last, int64_t n, T** ray_in /*x y z L M N i w opd*/,
                        T** rec /*8 x rows*n*/, T** grec /*8, entries may be null*/, T** gin /*8 out*/,
                        double* gparams /*n_surf*GP_COUNT, accumulated*/, char* err, int err_len,
                        double* gtab = nullptr /*n_surf*GT_PER_SURFACE, accumulated (polynomial families)*/) {
  PrepResult pr = prepare_table(*tab);
  if (!pr.error.empty()) { snprintf(err, err_len, "%s", pr.error.c_str()); return OLB_ERR_TABLE; }
  if (!pr.bwd_supported) { snprintf(err, err_len, "table outside the adjoint's scope"); return OLB_ERR_UNSUPPORTED; }
  if (pr.bwd_tables && !gtab) { snprintf(err, err_len, "polynomial-family table: gradient tables required"); return OLB_ERR_UNSUPPORTED; }
  const unsigned char* blob = sizeof(T) == 8 ? pr.blob_f64.data() : pr.blob_f32.data();
  const PrepHeader* H = reinterpret_cast<const PrepHeader*>(blob);
  const PrepSurface<T>* surf = reinterpret_cast<const PrepSurface<T>*>(blob + sizeof(PrepHeader));
  const T* pool = reinterpret_cast<const T*>(surf + H->n_surf);
  for (int64_t k = 0; k < n; ++k) {
    Adjoint<T> a{0, 0, 0, 0, 0, 0, 0, 0};
    for (int s = last - 1; s >= first; --s) {
      const int64_t off = (int64_t)(s - first) * n + k;
      if (grec[0]) a.x += grec[0][off];
      if (grec[1]) a.y += grec[1][off];
      if (grec[2]) a.z += grec[2][off];
      if (grec[3]) a.L += grec[3][off];
      if (grec[4]) a.M += grec[4][off];
      if (grec[5]) a.N += grec[5][off];
      if (grec[6]) a.i += grec[6][off];
      if (grec[7]) a.opd += grec[7][off];
      const PrepSurface<T>& S = surf[s];
      if (S.kind == OLB_GEOM_NOOP) continue;
      T pre[7];
      if (s == first) { for (int q = 0; q < 7; ++q) pre[q] = ray_in[q][k]; }
      else { for (int q = 0; q < 7; ++q) pre[q] = rec[q][off - n]; }
      T pg[GP_SCALARS] = {0}, r9[9] = {0};
      PolyAdj<T> pa{};
      surface_backward<T>(S, pool, pre[0], pre[1], pre[2], pre[3], pre[4], pre[5], pre[6], rec[0][off], rec[1][off],
                          rec[2][off], a, pg, (S.flags & OLB_SF_ROTATED) ? r9 : nullptr, 1, &pa);
      if (pa.active && gtab) {
        double* gS = gtab + (int64_t)s * GT_PER_SURFACE;
        double* gD = gS + GT_BLOCK;
        const bool tri = (S.flags & PSF_POLY_TRI) != 0;
        T xi = 1, xim = 0;
        for (int i = 0; i < S.poly_rows; ++i) {
          T yj = 1, yjm = 0;
          const int jmax = tri ? (S.poly_rows - 1 - i) : (S.poly_cols - 1);
          for (int j = 0; j <= jmax; ++j) {
            T vS, vD;
            poly_table_terms(pa, i, j, xi, xim, yj, yjm, vS, vD);
            gS[i * GT_DIM + j] += (double)vS;
            gD[i * GT_DIM + j] += (double)vD;
            yjm = yj; yj *= pa.yn;
          }
          xim = xi; xi *= pa.xn;
        }
      }
      for (int q = 0; q < GP_SCALARS; ++q) gparams[(int64_t)s * GP_COUNT + q] += (double)pg[q];
      for (int q = 0; q < 9; ++q) gparams[(int64_t)s * GP_COUNT + GP_R + q] += (double)r9[q];
    }
    gin[0][k] = a.x; gin[1][k] = a.y; gin[2][k] = a.z; gin[3][k] = a.L; gin[4][k] = a.M; gin[5][k] = a.N;
    gin[6][k] = a.i; gin[7][k] = a.opd;
  }
  return OLB_OK;
}

extern "C" {
int olbhc_backward_f64(const OlbTable* tab, int first, int last, int64_t n, double** ray_in, double** rec,
                       double** grec, double** gin, double* gparams, char* err, int err_len) {
  return run_backward<double>(tab, first, last, n, ray_in, rec, grec, gin, gparams, err, err_len);
}
int olbhc_backward_f32(const OlbTable* tab, int first, int last, int64_t n, float** ray_in, float** rec,
                       float** grec, float** gin, double* gparams, char* err, int err_len) {
  return run_backward<float>(tab, first, last, n, ray_in, rec, grec, gin, gparams, err, err_len);
}
int olbhc_gp_count() { return GP_COUNT; }
int olbhc_gt_per_surface() { return GT_PER_SURFACE; }
int olbhc_backward_tables_f64(const OlbTable* tab, int first, int last, int64_t n, double** ray_in, double** rec,
                              double** grec, double** gin, double* gparams, double* gtab, char* err, int err_len) {
  return run_backward<double>(tab, first, last, n, ray_in, rec, grec, gin, gparams, err, err_len, gtab);
}
int olbhc_backward_tables_f32(const OlbTable* tab, int first, int last, int64_t n, float** ray_in, float** rec,
                              float** grec, float** gin, double* gparams, double* gtab, char* err, int err_len) {
  return run_backward<float>(tab, first, last, n, ray_in, rec, grec, gin, gparams, err, err_len, gtab);
}
int olbhc_bwd_supported(const OlbTable* tab) {
  PrepResult pr = prepare_table(*tab);
  return pr.error.empty() && pr.bwd_supported ? 1 : 0;
}
// what olb_table_upload stores in OlbDeviceTable.bwd_supported (0, 1, or 2: table gradients) and .bwd_slots
// (PrepResult.total_gslots, the per-thread accumulator slots of the backward kernel); -1 on a table error
int olbhc_bwd_level(const OlbTable* tab) {
  PrepResult pr = prepare_table(*tab);
  return pr.error.empty() ? (pr.bwd_supported ? (pr.bwd_tables ? 2 : 1) : 0) : -1;
}
int olbhc_bwd_slots(const OlbTable* tab) {
  PrepResult pr = prepare_table(*tab);
  return pr.error.empty() ? pr.total_gslots : -1;
}
int olbhc_trace_f64(const OlbTable* tab, int first, int last, int64_t n, double** ray, double** rec, double** l0,
                    double* pmat, int* status, char* err, int err_len) {
  return run<double>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len);
}
int olbhc_trace_f32(const OlbTable* tab, int first, int last, int64_t n, float** ray, float** rec, float** l0,
                    float* pmat, int* status, char* err, int err_len) {
  return run<float>(tab, first, last, n, ray, rec, l0, pmat, status, err, err_len);
}
// intensity epilogue of the polarized kernels (olb_math.cuh::polarized_intensity) over n rays: pmat = [n][18],
// k = launch direction (3 arrays), i0, mode 1 (one state, ax / ay complex amplitudes) or 2 (unpolarized)
int olbhc_pol_intensity(int64_t n, const double* pmat, const double* kx, const double* ky, const double* kz,
                        const double* i0, int mode, const double* ax, const double* ay, double* out, int* status) {
  int st = 0;
  for (int64_t k = 0; k < n; ++k)
    out[k] = polarized_intensity<double>(pmat + k * 18, 1, kx[k], ky[k], kz[k], i0[k], mode, ax, ay, st);
  *status = st;
  return 0;
}
// wavefront epilogue (olb_math.cuh::wavefront_point) over n rays: fin = x y z L M N opd (fp64), ref = the 9
// doubles of WavefrontRef, out = opd_wv, pupil_x, pupil_y, pupil_z
int olbhc_wavefront(int64_t n, double** fin, const double* Px, const double* Py, const double* ref, double** out) {
  WavefrontRef w;
  w.c[0] = ref[0]; w.c[1] = ref[1]; w.c[2] = ref[2]; w.R = ref[3]; w.n_image = ref[4];
  w.tilt[0] = ref[5]; w.tilt[1] = ref[6]; w.opd_ref = ref[7]; w.inv_wl = ref[8];
  for (int64_t k = 0; k < n; ++k)
    wavefront_point(fin[0][k], fin[1][k], fin[2][k], fin[3][k], fin[4][k], fin[5][k], fin[6][k], Px[k], Py[k], w,
                    out[0][k], out[1][k], out[2][k], out[3][k]);
  return 0;
}
// host logic of the batched-systems upload (olb_prep.h::prepare_batch): copy system `b`'s prepared blob
// (which = 0: fp64, 1: fp32) into out; returns its size, or -1 on error (message in err)
int olbhc_batch_blob(const OlbTable* tmpl, const double* params, int n_systems, int b, int which, unsigned char* out,
                     int out_cap, unsigned* features, char* err, int err_len) {
  BatchPrep bp = prepare_batch(*tmpl, params, n_systems);
  if (!bp.error.empty()) { snprintf(err, err_len, "%s", bp.error.c_str()); return -1; }
  const int nb = which == 0 ? bp.bytes_f64 : bp.bytes_f32;
  if (b < 0 || b >= n_systems || nb > out_cap) { snprintf(err, err_len, "bad system index / buffer"); return -1; }
  const std::vector<unsigned char>& all = which == 0 ? bp.all64 : bp.all32;
  memcpy(out, all.data() + (size_t)b * nb, nb);
  *features = bp.features;
  return nb;
}
int olbhc_single_blob(const OlbTable* tab, int which, unsigned char* out, int out_cap, unsigned* features, char* err,
                      int err_len) {
  PrepResult pr = prepare_table(*tab);
  if (!pr.error.empty()) { snprintf(err, err_len, "%s", pr.error.c_str()); return -1; }
  const std::vector<unsigned char>& blob = which == 0 ? pr.blob_f64 : pr.blob_f32;
  if ((int)blob.size() > out_cap) { snprintf(err, err_len, "buffer too small"); return -1; }
  memcpy(out, blob.data(), blob.size());
  *features = pr.features;
  return (int)blob.size();
}
int olbhc_features(const OlbTable* tab) {
  PrepResult pr = prepare_table(*tab);
  return pr.error.empty() ? (int)pr.features : -1;
}

// FFT-PSF gridding (olb_fftpsf.cuh): the kernels' per-cell functions looped over the grid on the CPU
int olbhc_fft_pupil_f64(const double* opd, const double* inten, const int32_t* cell_ray, int32_t num_rays, int32_t grid,
                        double* pupil /* grid*grid*2 */) {
  const int32_t pad = (grid - num_rays) / 2;
  for (int32_t r = 0; r < grid; ++r)
    for (int32_t c = 0; c < grid; ++c) {
      double re, im;
      fft_pupil_cell<double>(r, c, num_rays, pad, cell_ray, opd, inten, re, im);
      pupil[2 * ((int64_t)r * grid + c)] = re;
      pupil[2 * ((int64_t)r * grid + c) + 1] = im;
    }
  return OLB_OK;
}
int olbhc_fft_pupil_f32(const float* opd, const float* inten, const int32_t* cell_ray, int32_t num_rays, int32_t grid,
                        float* pupil) {
  const int32_t pad = (grid - num_rays) / 2;
  for (int32_t r = 0; r < grid; ++r)
    for (int32_t c = 0; c < grid; ++c) {
      float re, im;
      fft_pupil_cell<float>(r, c, num_rays, pad, cell_ray, opd, inten, re, im);
      pupil[2 * ((int64_t)r * grid + c)] = re;
      pupil[2 * ((int64_t)r * grid + c) + 1] = im;
    }
  return OLB_OK;
}
int olbhc_fft_psf_accumulate_f64(const double* amp, int32_t grid, int32_t first, int32_t last, double div, double mul,
                                 double* psf) {
  for (int32_t r = 0; r < grid; ++r)
    for (int32_t c = 0; c < grid; ++c) {
      const int64_t k = (int64_t)r * grid + c;
      const int64_t o = (int64_t)fftshift_index(r, grid) * grid + fftshift_index(c, grid);
      psf[o] = fft_psf_cell<double>(first ? 0.0 : psf[o], amp[2 * k], amp[2 * k + 1], first != 0, last != 0, div, mul);
    }
  return OLB_OK;
}
}
