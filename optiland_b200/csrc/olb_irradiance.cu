// olb_irradiance.cu -- incoherent irradiance binning (IncoherentIrradiance, optiland/analysis/irradiance.py:265-353),
// sm_90a.  Per-ray arithmetic and its semantics: olb_irradiance.cuh and include/olb.h (OlbIrradiance).
//
// One streaming pass over the final ray state: 12 B (fp32) / 24 B (fp64) read per ray in an unrotated frame, 16 / 32 B
// when z is needed.  Two ways to accumulate, chosen from the grid size and the ray count (irr_use_shared):
//   * shared: each CTA keeps a private fp64 histogram in shared memory (128 KiB for the default 128 x 128 grid) and
//     flushes its non-zero bins to global memory with one fp64 atomic each.  It is taken only with >= 256 rays per bin
//     and the grid is sized to at least one ray per bin of each private copy, so zeroing and flushing the copies never
//     costs more than the binning.
//   * global: one fp64 reduction to global memory per kept ray (native RED.ADD.F64; the shared path's fp64 atomic is a
//     compare-and-swap loop): fewer rays per bin, and grids whose histogram does not fit in shared memory.
// On both, lanes of a warp that hit the same bin are summed before their atomic (irr_add).
#include <cuda_runtime.h>
#include <stdint.h>

#include <mutex>
#include <string>
#include <unordered_map>

#include "../../include/olb.h"
#include "olb_irradiance.cuh"

namespace olb {
int fail_psf(int code, const char* msg);   // olb_trace.cu
void count_launch();

static constexpr int IRR_BLOCK_SHARED = 1024;
static constexpr int IRR_BLOCK_GLOBAL = 256;
// Largest grid binned through per-CTA shared-memory copies: 27 x 1024 doubles = 216 KiB, inside the 227 KiB a CTA
// may opt into on sm_90.
static constexpr int64_t IRR_SHARED_MAX_BINS = 27 * 1024;

template <typename T>
struct IrrArgs {
  const T* x; const T* y; const T* z; const T* i;
  int64_t n;
  IrrFrame frame;
  const double* xe; const double* ye;
  int32_t nx, ny;
  double x_inv, y_inv;
  double* hist;
};

template <typename T>
__device__ __forceinline__ int64_t irr_bin_of(const IrrArgs<T>& a, int64_t r, double& w) {
  const T z = a.frame.affine ? a.z[r] : (T)0;
  const T p = a.i[r];
  w = (double)p;
  return irr_ray_bin<T>(a.x[r], a.y[r], z, p, a.frame, a.xe, a.nx, a.x_inv, a.ye, a.ny, a.y_inv);
}

// Add w into h[b] for every lane with b >= 0.  Lanes of the warp that hit the same bin first sum their weights
// (__match_any_sync groups them; a log2-step tree over each group's ranks) and one lane per group issues the atomic:
// a focused beam sends whole warps to one bin, which otherwise serialises 32 atomics on one address (on an H100, 10^7
// rays into four bins: 0.67 ms -> 0.11 ms on the shared path, 6.4 ms -> 0.74 ms on the global path).  The grouping only
// runs when neighbouring lanes collide, which costs a uniform spread at most ~5 %.  Needs the whole warp converged (the
// callers' loops keep every lane iterating together).
__device__ __forceinline__ void irr_add(double* h, int64_t b, double w) {
  constexpr unsigned FULL = 0xffffffffu;
  const unsigned lane = threadIdx.x & 31u;
  // cheap screen first: grouping only pays when lanes collide, and then neighbouring lanes do too
  const long long below = __shfl_up_sync(FULL, (long long)b, 1);
  if (!__any_sync(FULL, lane > 0 && b >= 0 && b == below)) {
    if (b >= 0) atomicAdd(&h[b], w);
    return;
  }
  const unsigned peers = __match_any_sync(FULL, (unsigned long long)b);
  unsigned higher = peers & (0xfffffffeu << lane);          // peers on higher lanes, not yet folded in
  unsigned rank = __popc(peers & ((1u << lane) - 1u));      // position among the peers
  while (__any_sync(FULL, higher)) {
    const int next = __ffs(higher);                         // 1-based lane of the next higher peer, 0: none
    const double t = __shfl_sync(FULL, w, next ? next - 1 : (int)lane);
    if (next) w += t;
    higher &= ~__ballot_sync(FULL, rank & 1u);              // odd ranks have handed their partial sums on
    rank >>= 1;
  }
  if (b >= 0 && lane == (unsigned)(__ffs(peers) - 1)) atomicAdd(&h[b], w);
}

// One pass over the rays in warp-uniform steps (every lane runs the same number of iterations, as irr_add needs).
template <typename T>
__device__ __forceinline__ void irr_bin_all(const IrrArgs<T>& a, double* h) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t base = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < a.n; base += stride) {
    const int64_t r = base + (threadIdx.x & 31u);
    double w = 0.0;
    const int64_t b = r < a.n ? irr_bin_of(a, r, w) : -1;
    irr_add(h, b, w);
  }
}

template <typename T>
__global__ void __launch_bounds__(IRR_BLOCK_SHARED) irradiance_shared_kernel(const __grid_constant__ IrrArgs<T> a) {
  extern __shared__ double s_hist[];
  const int32_t nb = a.nx * a.ny;
  for (int32_t b = threadIdx.x; b < nb; b += blockDim.x) s_hist[b] = 0.0;
  __syncthreads();
  irr_bin_all<T>(a, s_hist);
  __syncthreads();
  for (int32_t b = threadIdx.x; b < nb; b += blockDim.x) {
    const double v = s_hist[b];
    if (v != 0.0) atomicAdd(&a.hist[b], v);
  }
}

template <typename T>
__global__ void __launch_bounds__(IRR_BLOCK_GLOBAL) irradiance_global_kernel(const __grid_constant__ IrrArgs<T> a) {
  irr_bin_all<T>(a, a.hist);
}

// SMs of the current device; a failed query leaves its error for the launch that follows to report
static int64_t irr_sm_count() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return 1;
  return n > 0 ? n : 1;
}

static bool irr_edges_ok(const double* e, int32_t n) {
  for (int32_t k = 0; k <= n; ++k)
    if (!isfinite(e[k]) || (k > 0 && !(e[k] > e[k - 1]))) return false;
  return true;
}

// The path a call with nb bins and n rays takes (OLB_IRR_PATH_AUTO): shared-memory copies pay once there are >= 256
// rays per bin.  Measured on an H100 (kernel time, both paths forced, fp32 and fp64): at 128 x 128 the global path wins
// at 10^6 rays (61 per bin; 18 vs 30 us), the two are within 7 % at 3 x 10^6 (183 per bin), the shared path wins at 10^7
// (610 per bin; 150 vs 161 us); at 32 x 32 it wins from 3 x 10^5 rays (293 per bin; 9 vs 19 us) and by 5x at 10^7; at
// 160 x 160 and 10^7 rays (390 per bin) they tie.  scripts/bench_irradiance.py times both paths on its workloads.
static bool irr_use_shared(int64_t nb, int64_t n) { return nb <= IRR_SHARED_MAX_BINS && n >= 256 * nb; }

// Resident CTAs per SM of the shared-path kernel for a histogram of nb bins, cached per device and nb (the opt-in
// attribute is set once per device at the largest histogram).  0 on a failed query, whose error the caller reports.
template <typename T>
static int shared_ctas_per_sm(int64_t nb, cudaError_t& e) {
  static std::mutex mu;
  static std::unordered_map<int64_t, int> cache;   // (device << 32) | nb -> CTAs per SM; nb = -1: attribute set
  int dev = 0;
  if ((e = cudaGetDevice(&dev)) != cudaSuccess) return 0;
  std::lock_guard<std::mutex> lock(mu);
  const int64_t key = ((int64_t)dev << 32) | nb, attr_key = ((int64_t)dev << 32) | 0xffffffffLL;
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  if (!cache.count(attr_key)) {
    e = cudaFuncSetAttribute(irradiance_shared_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)(IRR_SHARED_MAX_BINS * sizeof(double)));
    if (e != cudaSuccess) return 0;
    cache[attr_key] = 1;
  }
  int per_sm = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, irradiance_shared_kernel<T>, IRR_BLOCK_SHARED,
                                                    (size_t)nb * sizeof(double));
  if (e != cudaSuccess) return 0;
  cache[key] = per_sm;
  return per_sm;
}

template <typename T>
static cudaError_t launch_shared(const IrrArgs<T>& a, int64_t nb, cudaStream_t st) {
  cudaError_t e = cudaSuccess;
  const int per_sm = shared_ctas_per_sm<T>(nb, e);
  if (e != cudaSuccess) return e;
  if (per_sm < 1) return cudaErrorInvalidConfiguration;
  // at least max(nb, 4 rays per thread) rays per CTA: zeroing and flushing a private copy costs ~ one pass over it
  const int64_t per_cta = nb > 4 * IRR_BLOCK_SHARED ? nb : 4 * IRR_BLOCK_SHARED;
  int64_t ctas = (a.n + per_cta - 1) / per_cta;
  if (ctas > per_sm * irr_sm_count()) ctas = per_sm * irr_sm_count();
  irradiance_shared_kernel<T><<<(unsigned)ctas, IRR_BLOCK_SHARED, (size_t)nb * sizeof(double), st>>>(a);
  return cudaGetLastError();
}

template <typename T>
static cudaError_t launch_global(const IrrArgs<T>& a, cudaStream_t st) {
  int64_t ctas = (a.n + IRR_BLOCK_GLOBAL - 1) / IRR_BLOCK_GLOBAL;
  if (ctas > 8 * irr_sm_count()) ctas = 8 * irr_sm_count();
  irradiance_global_kernel<T><<<(unsigned)ctas, IRR_BLOCK_GLOBAL, 0, st>>>(a);
  return cudaGetLastError();
}

template <typename T>
static int irradiance_impl(const OlbIrradiance* c, void* stream, const char* name) {
  const std::string who(name);
  if (!c) return fail_psf(OLB_ERR_INVALID_ARG, (who + ": call is NULL").c_str());
  if (c->frame != OLB_IRR_FRAME_TRANSLATE && c->frame != OLB_IRR_FRAME_AFFINE)
    return fail_psf(OLB_ERR_INVALID_ARG, (who + ": frame must be OLB_IRR_FRAME_TRANSLATE or OLB_IRR_FRAME_AFFINE").c_str());
  if (!c->x || !c->y || !c->i || (c->frame == OLB_IRR_FRAME_AFFINE && !c->z) || !c->x_edges || !c->y_edges || !c->edges ||
      !c->hist)
    return fail_psf(OLB_ERR_INVALID_ARG, (who + ": NULL array").c_str());
  if (c->n_rays < 0) return fail_psf(OLB_ERR_INVALID_ARG, (who + ": n_rays < 0").c_str());
  if (c->nx < 1 || c->ny < 1) return fail_psf(OLB_ERR_INVALID_ARG, (who + ": nx and ny must be >= 1").c_str());
  if (c->path != OLB_IRR_PATH_AUTO && c->path != OLB_IRR_PATH_SHARED && c->path != OLB_IRR_PATH_GLOBAL)
    return fail_psf(OLB_ERR_INVALID_ARG, (who + ": path must be OLB_IRR_PATH_AUTO, _SHARED or _GLOBAL").c_str());
  if (c->path == OLB_IRR_PATH_SHARED && (int64_t)c->nx * c->ny > IRR_SHARED_MAX_BINS)
    return fail_psf(OLB_ERR_INVALID_ARG, (who + ": OLB_IRR_PATH_SHARED needs nx * ny <= 27648").c_str());
  if ((int64_t)c->nx * c->ny > INT32_MAX) return fail_psf(OLB_ERR_INVALID_ARG, (who + ": nx * ny too large").c_str());
  if (!irr_edges_ok(c->x_edges, c->nx))
    return fail_psf(OLB_ERR_INVALID_ARG, (who + ": x_edges must be finite and strictly increasing").c_str());
  if (!irr_edges_ok(c->y_edges, c->ny))
    return fail_psf(OLB_ERR_INVALID_ARG, (who + ": y_edges must be finite and strictly increasing").c_str());
  if (c->n_rays == 0) return OLB_OK;

  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemcpyAsync(c->edges, c->x_edges, (size_t)(c->nx + 1) * sizeof(double), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(c->edges + c->nx + 1, c->y_edges, (size_t)(c->ny + 1) * sizeof(double), cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) return fail_psf(OLB_ERR_CUDA, (who + ": edge upload: " + cudaGetErrorString(e)).c_str());

  IrrArgs<T> a;
  a.x = (const T*)c->x; a.y = (const T*)c->y; a.z = (const T*)c->z; a.i = (const T*)c->i;
  a.n = c->n_rays;
  a.frame.affine = c->frame == OLB_IRR_FRAME_AFFINE;
  for (int k = 0; k < 3; ++k) a.frame.t[k] = c->t[k];
  for (int k = 0; k < 9; ++k) a.frame.R[k] = a.frame.affine ? c->R[k] : (k % 4 == 0 ? 1.0 : 0.0);
  a.xe = c->edges; a.ye = c->edges + c->nx + 1;
  a.nx = c->nx; a.ny = c->ny;
  a.x_inv = c->nx / (c->x_edges[c->nx] - c->x_edges[0]);
  a.y_inv = c->ny / (c->y_edges[c->ny] - c->y_edges[0]);
  a.hist = c->hist;

  const int64_t nb = (int64_t)c->nx * c->ny;
  const int32_t want = c->path;
  const bool shared = want == OLB_IRR_PATH_SHARED || (want == OLB_IRR_PATH_AUTO && irr_use_shared(nb, c->n_rays));
  e = shared ? launch_shared<T>(a, nb, st) : launch_global<T>(a, st);
  if (e != cudaSuccess) return fail_psf(OLB_ERR_CUDA, (who + ": " + cudaGetErrorString(e)).c_str());
  count_launch();
  return OLB_OK;
}

}  // namespace olb

extern "C" int olb_irradiance_f32(const OlbIrradiance* call, void* stream) {
  return olb::irradiance_impl<float>(call, stream, "olb_irradiance_f32");
}
extern "C" int olb_irradiance_f64(const OlbIrradiance* call, void* stream) {
  return olb::irradiance_impl<double>(call, stream, "olb_irradiance_f64");
}
