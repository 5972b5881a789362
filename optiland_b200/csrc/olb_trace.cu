// olb_trace.cu -- sm_90a trace kernel + the C ABI of include/olb.h.
//
// Forward: ONE kernel walks the WHOLE surface list for a tile of rays: the ray state lives in
// registers from launch state to image surface, the prepared surface table lives in shared
// memory (one TMA bulk copy per CTA), and the only HBM traffic is the algorithmic minimum --
// 8 coalesced vector loads per ray (2 in pupil-launch mode) and 8 streaming vector stores per
// ray per recorded surface (SURVEY.md section 8d).  The reference does the same work with ~190
// eager element-wise launches per surface (SURVEY.md section 1).  Optional in-kernel stages:
// launch-state generation from pupil coordinates (8f-1), polarization matrices, spot / OPD
// moments and the wavefront (OPD-map) epilogue (8f-2), many systems per launch (8f-4: blockIdx.y =
// system, each CTA stages its own system's table).  Backward: one adjoint kernel (trace_bwd_kernel).
//
// No tensor cores: there is no contraction on this path.  The roofline is HBM.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <atomic>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/olb.h"
#include "olb_math.cuh"
#include "olb_bsdf.cuh"
#include "olb_aim.cuh"
#include "olb_prep.h"

namespace olb {

static constexpr int BLOCK = 256;
// Minimum resident CTAs per SM asked of ptxas: 16 bytes of ray state per access (float4 /
// double2) -> 2 CTAs (<= 128 registers), narrower variants -> 3 CTAs (<= 85 registers).
template <typename T, int RPT, uint32_t FEAT> struct MinBlocks {
  // polarized: the P matrix lives in shared memory, so both precisions fit 2 CTAs per SM (<= 128 registers)
  static constexpr int v = (FEAT & 8u) ? 2 : ((sizeof(T) * RPT <= 8) ? 3 : 2);
};
// Host-buffer pipeline: chunks in flight (H2D of one overlaps kernel / D2H of the others).
static constexpr int HOST_SLOTS = 3;

static thread_local std::string g_last_error;
static std::atomic<int64_t> g_launches{0};

static int fail(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}
int fail_psf(int code, const char* msg) { return fail(code, msg); }   // used by olb_psf.cu
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
#define OLB_CUDA(call)                                                                    \
  do {                                                                                    \
    cudaError_t e__ = (call);                                                             \
    if (e__ != cudaSuccess)                                                               \
      return fail(OLB_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e__));     \
  } while (0)

// Device workspace layout: [64-byte pad][blob f64][blob f32], each 16-byte aligned.
static constexpr uint32_t WS_MAGIC = 0x4f4c4231u;  // "OLB1"

struct TraceArgs {
  const unsigned char* blob;  // prepared table for this element type (device)
  int32_t blob_bytes;
  int32_t first, last;
  uint32_t tflags;
  int64_t n_rays;
  int64_t rec_stride;
  void* x; void* y; void* z; void* L; void* M; void* N; void* i; void* w; void* opd;
  void* L0; void* M0; void* N0; void* p;
  void* rx; void* ry; void* rz; void* rL; void* rM; void* rN; void* ri; void* ropd;
  int32_t* status;
  // launch state from pupil coordinates (OlbPupilLaunch) when px != nullptr
  const void* px; const void* py;
  double lo0[3], los[2], lt0[3], lts[2], linten;
  // per-ray field coordinates (trace_generic): origin / target offsets lof * g(H), ltf * g(H)
  const void* hx; const void* hy;
  int32_t fmode; int32_t n_vig;
  double farg, lof[2], ltf[2];
  int32_t vig_power; int32_t vpad;
  double vig[OLB_MAX_VIG_FIELDS][4];   // per-ray vignetting factors: nearest defined field (Hx, Hy, vx, vy)
  // fused moments epilogue (OLB_TF_MOMENTS)
  double* moments;
  double mcx, mcy;
  // batched systems (OlbTraceCall.rays_per_system): blockIdx.y = system, its table at blob + y * blob_stride, its rays
  // are the segment [y * sys_rays, (y+1) * sys_rays); shared_in: every system reads the SAME sys_rays inputs
  int64_t sys_rays;
  int32_t blob_stride;
  int32_t shared_in;
  // wavefront epilogue (OlbTraceCall.wavefront_out) when wf_opd != nullptr
  void* wf_opd; void* wf_px; void* wf_py; void* wf_pz; void* wf_i;
  WavefrontRef wf;
  // polarized intensity epilogue (OlbPolarization): 0 off, 1 one polarized state, 2 unpolarized
  int32_t pol_mode; int32_t pol_pad;
  double pol_ax[2], pol_ay[2];     // complex amplitudes Ex e^{i phase_x}, Ey e^{i phase_y}
  void* pol_i;                     // optional separate output of the updated intensity
  // BSDF scatter draws (FEAT_BSDF kernels): ray index = ray0 + index in this call's arrays, Philox counter word
  int64_t ray0;
  uint32_t rng_stream; int32_t rng_pad;
};

// Shared-memory slots per thread of a polarized kernel: the P matrix (18) + launch direction (3) + launch intensity
constexpr int POL_SLOTS = 22;

// ---- vector access helpers -------------------------------------------------------------
template <typename T, int RPT> struct Vec;
template <> struct Vec<float, 4> { using type = float4; };
template <> struct Vec<float, 2> { using type = float2; };
template <> struct Vec<double, 2> { using type = double2; };
template <> struct Vec<float, 1> { using type = float; };
template <> struct Vec<double, 1> { using type = double; };

template <typename T, int RPT>
__device__ __forceinline__ void load_rays(const T* __restrict__ p, int64_t base, int valid, T (&v)[RPT]) {
  if constexpr (RPT == 1) {
    v[0] = __ldcs(p + base);
  } else {
    if (valid == RPT) {
      using V = typename Vec<T, RPT>::type;
      V q = __ldcs(reinterpret_cast<const V*>(p + base));
      const T* e = reinterpret_cast<const T*>(&q);
#pragma unroll
      for (int k = 0; k < RPT; ++k) v[k] = e[k];
    } else {
#pragma unroll
      for (int k = 0; k < RPT; ++k) v[k] = k < valid ? __ldcs(p + base + k) : (T)0;
    }
  }
}
template <typename T, int RPT>
__device__ __forceinline__ void store_rays(T* __restrict__ p, int64_t base, int valid, const T (&v)[RPT]) {
  if constexpr (RPT == 1) {
    __stcs(p + base, v[0]);
  } else {
    if (valid == RPT) {
      using V = typename Vec<T, RPT>::type;
      V q;
      T* e = reinterpret_cast<T*>(&q);
#pragma unroll
      for (int k = 0; k < RPT; ++k) e[k] = v[k];
      __stcs(reinterpret_cast<V*>(p + base), q);
    } else {
#pragma unroll
      for (int k = 0; k < RPT; ++k)
        if (k < valid) __stcs(p + base + k, v[k]);
    }
  }
}

__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// ---- TMA bulk copy of the prepared table into shared memory ------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void stage_table(unsigned char* smem, const unsigned char* gsrc, uint32_t bytes,
                                            uint64_t* bar) {
  const uint32_t bar_a = smem_u32(bar);
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes) : "memory");
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(smem)),
        "l"(gsrc), "r"(bytes), "r"(bar_a)
        : "memory");
  }
  // every thread waits for the bytes to land (phase 0)
  uint32_t done = 0;
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar_a)
        : "memory");
  }
}

// ---- the kernel -----------------------------------------------------------------------------
template <typename T, int RPT, uint32_t FEAT>
__global__ void __launch_bounds__(BLOCK, (MinBlocks<T, RPT, FEAT>::v)) trace_kernel(const __grid_constant__ TraceArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem);
  unsigned char* tab = smem + 16;
  const int sys = blockIdx.y;                                   // 0 unless batched
  stage_table(tab, a.blob + (size_t)sys * (size_t)a.blob_stride, (uint32_t)a.blob_bytes, bar);

  const PrepHeader* H = reinterpret_cast<const PrepHeader*>(tab);
  const PrepSurface<T>* surf = reinterpret_cast<const PrepSurface<T>*>(tab + sizeof(PrepHeader));
  const T* pool = reinterpret_cast<const T*>(surf + H->n_surf);
  const int n_wl = H->n_wl;
  const T* wl = pool + H->pad[0];
  // Polarized kernels keep each ray's P matrix (and its launch direction / intensity for the intensity epilogue)
  // in shared memory, [slot][thread]: conflict-free, and the 18 + 4 values are not live registers across the
  // geometry step (the register-resident form needed 204 registers in fp64: one CTA per SM).
  T* Psm = reinterpret_cast<T*>(tab + (((size_t)a.blob_bytes + 15) & ~size_t(15))) + threadIdx.x;

  const int64_t n = a.sys_rays > 0 ? a.sys_rays : a.n_rays;     // rays of THIS system
  const int64_t seg = (int64_t)sys * n;                         // where its outputs start
  const int64_t per_tile = (int64_t)BLOCK * RPT;
  const int64_t n_tiles = (n + per_tile - 1) / per_tile;
  const int first = a.first, last = a.last;
  int status = 0;
  double mom[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // OLB_TF_MOMENTS: per-thread partial sums

  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t local = (tile * BLOCK + threadIdx.x) * RPT;
    if (local >= n) continue;
    const int valid = (n - local) >= RPT ? RPT : (int)(n - local);
    const int64_t base = seg + local;                           // output index
    const int64_t bin = a.shared_in ? local : base;             // input index

    Ray<T> r[RPT];
    {
      T v[RPT];
      if (a.px != nullptr) {
        // launch state generated from the pupil point: 2 loads instead of 8
        T pv[RPT];
        load_rays<T, RPT>((const T*)a.px, bin, valid, pv);
        load_rays<T, RPT>((const T*)a.py, bin, valid, v);
        const T o0[3] = {(T)a.lo0[0], (T)a.lo0[1], (T)a.lo0[2]}, os[2] = {(T)a.los[0], (T)a.los[1]};
        const T t0[3] = {(T)a.lt0[0], (T)a.lt0[1], (T)a.lt0[2]}, ts[2] = {(T)a.lts[0], (T)a.lts[1]};
        if (a.hx != nullptr) {
          // field point per ray: angle fields move origin (and target) by tan(H * max_field), object heights by H
          T hxv[RPT], hyv[RPT];
          load_rays<T, RPT>((const T*)a.hx, bin, valid, hxv);
          load_rays<T, RPT>((const T*)a.hy, bin, valid, hyv);
          if (a.n_vig > 0) {
            // FieldGroup.get_vig_factor: nearest defined field; the pupil point shrinks by (1 - vx, 1 - vy)
#pragma unroll
            for (int k = 0; k < RPT; ++k) {
              int best = 0;
              double bd = 1e300;
              for (int j = 0; j < a.n_vig; ++j) {
                const double dx = (double)hxv[k] - a.vig[j][0], dy = (double)hyv[k] - a.vig[j][1];
                const double d2 = dx * dx + dy * dy;
                if (d2 < bd) { bd = d2; best = j; }
              }
              const T sx = (T)1 - (T)a.vig[best][2], sy = (T)1 - (T)a.vig[best][3];
              for (int q = 0; q < a.vig_power; ++q) { pv[k] = pv[k] * sx; v[k] = v[k] * sy; }
            }
          }
#pragma unroll
          for (int k = 0; k < RPT; ++k) {
            // fp64 tangent for both element types: a field angle feeds a lever arm of hundreds of mm
            const double gx = a.fmode == 1 ? tan(a.farg * (double)hxv[k]) : (double)hxv[k];
            const double gy = a.fmode == 1 ? tan(a.farg * (double)hyv[k]) : (double)hyv[k];
            pupil_launch<T>(r[k], pv[k], v[k], o0, os, t0, ts, (T)a.linten, (T)(a.lof[0] * gx), (T)(a.lof[1] * gy),
                            (T)(a.ltf[0] * gx), (T)(a.ltf[1] * gy));
          }
        } else {
#pragma unroll
          for (int k = 0; k < RPT; ++k) pupil_launch<T>(r[k], pv[k], v[k], o0, os, t0, ts, (T)a.linten);
        }
      } else {
      load_rays<T, RPT>((const T*)a.x, bin, valid, v);
#pragma unroll
      for (int k = 0; k < RPT; ++k) r[k].x = v[k];
      load_rays<T, RPT>((const T*)a.y, bin, valid, v);
#pragma unroll
      for (int k = 0; k < RPT; ++k) r[k].y = v[k];
      load_rays<T, RPT>((const T*)a.z, bin, valid, v);
#pragma unroll
      for (int k = 0; k < RPT; ++k) r[k].z = v[k];
      load_rays<T, RPT>((const T*)a.L, bin, valid, v);
#pragma unroll
      for (int k = 0; k < RPT; ++k) r[k].L = v[k];
      load_rays<T, RPT>((const T*)a.M, bin, valid, v);
#pragma unroll
      for (int k = 0; k < RPT; ++k) r[k].M = v[k];
      load_rays<T, RPT>((const T*)a.N, bin, valid, v);
#pragma unroll
      for (int k = 0; k < RPT; ++k) r[k].N = v[k];
      load_rays<T, RPT>((const T*)a.i, bin, valid, v);
#pragma unroll
      for (int k = 0; k < RPT; ++k) r[k].i = v[k];
      load_rays<T, RPT>((const T*)a.opd, bin, valid, v);
#pragma unroll
      for (int k = 0; k < RPT; ++k) r[k].opd = v[k];
      }
#pragma unroll
      for (int k = 0; k < RPT; ++k) { r[k].opd_lo = 0; r[k].widx = 0; r[k].L0 = r[k].M0 = r[k].N0 = 0; }
      if constexpr ((FEAT & FEAT_BSDF) != 0) {
#pragma unroll
        for (int k = 0; k < RPT; ++k) { r[k].id = (uint64_t)(a.ray0 + base + k); r[k].stream = a.rng_stream; }
      }
      if (n_wl > 1) {
        load_rays<T, RPT>((const T*)a.w, bin, valid, v);
#pragma unroll
        for (int k = 0; k < RPT; ++k) {
          int idx = -1;
          for (int j = 0; j < n_wl; ++j)
            if (v[k] == wl[j]) idx = j;
          r[k].widx = idx;
        }
      }
    }

    if constexpr ((FEAT & FEAT_POL) != 0) {
      static_assert(RPT == 1, "polarized kernels process one ray per thread");
      if (a.tflags & OLB_TF_POL_IDENTITY) {
#pragma unroll
        for (int q = 0; q < 18; ++q) Psm[q * BLOCK] = (q == 0 || q == 8 || q == 16) ? (T)1 : (T)0;
      } else {
        using V2 = typename Vec<T, 2>::type;
        const V2* src = reinterpret_cast<const V2*>((const T*)a.p + base * 18);
#pragma unroll
        for (int q = 0; q < 9; ++q) {
          V2 v = __ldcs(src + q);
          Psm[(2 * q) * BLOCK] = v.x; Psm[(2 * q + 1) * BLOCK] = v.y;
        }
      }
      if (a.pol_mode != 0) {   // what update_intensity needs from the LAUNCH state (polarized_rays.py:51-55)
        Psm[18 * BLOCK] = r[0].L; Psm[19 * BLOCK] = r[0].M; Psm[20 * BLOCK] = r[0].N; Psm[21 * BLOCK] = r[0].i;
      }
    }

    // Pull the NEXT tile's launch state into L2 while this tile computes (no registers held):
    // the first loads of the next iteration then see L2 latency instead of HBM latency.
    {
      const int64_t nb = bin + (int64_t)gridDim.x * per_tile;
      if (a.sys_rays > 0) {
        // batched: one tile per CTA, nothing to prefetch
      } else if (a.px != nullptr) {
        if (nb + RPT <= n && (threadIdx.x * RPT * (int)sizeof(T)) % 32 == 0) {
          prefetch_l2((const T*)a.px + nb); prefetch_l2((const T*)a.py + nb);
        }
      } else if (nb + RPT <= n && (threadIdx.x * RPT * (int)sizeof(T)) % 32 == 0) {
        prefetch_l2((const T*)a.x + nb); prefetch_l2((const T*)a.y + nb); prefetch_l2((const T*)a.z + nb);
        prefetch_l2((const T*)a.L + nb); prefetch_l2((const T*)a.M + nb); prefetch_l2((const T*)a.N + nb);
        prefetch_l2((const T*)a.i + nb); prefetch_l2((const T*)a.opd + nb);
        if (n_wl > 1) prefetch_l2((const T*)a.w + nb);
      }
    }

    bool have_frame = false;  // false: registers hold GLOBAL coordinates
    T gx[RPT], gy[RPT], gz[RPT], gL[RPT], gM[RPT], gN[RPT];
#pragma unroll
    for (int k = 0; k < RPT; ++k) { gx[k] = r[k].x; gy[k] = r[k].y; gz[k] = r[k].z; gL[k] = r[k].L; gM[k] = r[k].M; gN[k] = r[k].N; }

    for (int s = first; s < last; ++s) {
      const PrepSurface<T>& S = surf[s];
      const bool noop = S.kind == OLB_GEOM_NOOP;
      if (!noop) {
        // geometry dispatch ONCE per surface (warp-uniform), outside the per-ray loop
        const bool fg = !have_frame;
        if (S.kind == OLB_GEOM_PLANE) {
#pragma unroll
          for (int k = 0; k < RPT; ++k) surface_step_k<T, FEAT, KIND_PLANE>(r[k], S, pool, fg, status, Psm, BLOCK);
        } else if (S.kind == OLB_GEOM_STANDARD) {
#pragma unroll
          for (int k = 0; k < RPT; ++k) surface_step_k<T, FEAT, KIND_CONIC>(r[k], S, pool, fg, status, Psm, BLOCK);
        } else if constexpr ((FEAT & FEAT_GRID) != 0) {
          // grid-sag tables run the general kernel (FEAT_FREEFORM): the grid loop beside the one generic Newton loop
          if (S.kind == OLB_GEOM_GRID_SAG) {
#pragma unroll
            for (int k = 0; k < RPT; ++k) surface_step_k<T, FEAT, KIND_GRID>(r[k], S, pool, fg, status, Psm, BLOCK);
          } else {
#pragma unroll
            for (int k = 0; k < RPT; ++k) surface_step_k<T, FEAT, KIND_NEWTON>(r[k], S, pool, fg, status, Psm, BLOCK);
          }
        } else if constexpr ((FEAT & FEAT_NEWTON) != 0) {
          // (the launcher gives Newton tables RPT <= 2, so the unrolled bodies stay inside the I-cache.)
          // Asphere-only tables (no FEAT_FREEFORM) run the fused sag + slope loop; tables with a polynomial-family
          // surface run ONE generic loop for all their Newton surfaces.
          if constexpr ((FEAT & FEAT_FREEFORM) != 0) {
#pragma unroll
            for (int k = 0; k < RPT; ++k) surface_step_k<T, FEAT, KIND_NEWTON>(r[k], S, pool, fg, status, Psm, BLOCK);
          } else {
#pragma unroll
            for (int k = 0; k < RPT; ++k) surface_step_k<T, FEAT, KIND_ASPHERE>(r[k], S, pool, fg, status, Psm, BLOCK);
          }
        }
        have_frame = true;
      }
      const bool record = a.rx != nullptr && !(S.flags & OLB_SF_NORECORD);
      if (record || s == last - 1) {
        if (!noop) {
#pragma unroll
          for (int k = 0; k < RPT; ++k) to_global<T, FEAT>(r[k], S, gx[k], gy[k], gz[k], gL[k], gM[k], gN[k]);
        }
      }
      if (record) {
        const int64_t off = (int64_t)(s - first) * a.rec_stride + base;
        T v[RPT];
        store_rays<T, RPT>((T*)a.rx, off, valid, gx);
        store_rays<T, RPT>((T*)a.ry, off, valid, gy);
        store_rays<T, RPT>((T*)a.rz, off, valid, gz);
        store_rays<T, RPT>((T*)a.rL, off, valid, gL);
        store_rays<T, RPT>((T*)a.rM, off, valid, gM);
        store_rays<T, RPT>((T*)a.rN, off, valid, gN);
#pragma unroll
        for (int k = 0; k < RPT; ++k) v[k] = r[k].i;
        store_rays<T, RPT>((T*)a.ri, off, valid, v);
#pragma unroll
        for (int k = 0; k < RPT; ++k) v[k] = opd_value(r[k]);
        store_rays<T, RPT>((T*)a.ropd, off, valid, v);
      }
    }

    if (a.tflags & OLB_TF_MOMENTS) {
      // intercepts on the LAST traced surface: its local frame (r.x, r.y) with the mask i > 0 and finite (what
      // SpotDiagram transforms to and keeps), or -- OLB_TF_MOMENTS_GLOBAL / _ALL -- global coordinates / every ray
      // (what the rms_spot_size operand averages: a NaN ray then makes the sums NaN, as in the reference)
      const bool glob = (a.tflags & OLB_TF_MOMENTS_GLOBAL) != 0, all = (a.tflags & OLB_TF_MOMENTS_ALL) != 0;
#pragma unroll
      for (int k = 0; k < RPT; ++k) {
        if (k >= valid) continue;
        const double dx = (double)(glob ? gx[k] : r[k].x) - a.mcx, dy = (double)(glob ? gy[k] : r[k].y) - a.mcy;
        const double ii = (double)r[k].i, oo = (double)opd_value(r[k]);
        const bool finite = dx - dx == 0 && dy - dy == 0;
        if (all || (ii > 0 && finite)) {
          mom[0] += 1.0; mom[1] += dx; mom[2] += dy; mom[3] += dx * dx + dy * dy; mom[4] += ii;
          mom[5] += oo; mom[6] += oo * oo;
        } else if (ii > 0) {
          mom[7] += 1.0;          // kept by the reference's mask (i > 0) but not finite: its statistics are NaN
        }
      }
    }
    if constexpr ((FEAT & FEAT_POL) != 0) {
      if (a.pol_mode != 0) {
        // PolarizedRays.update_intensity on the final P matrix; the record rows above keep the geometric intensity
        const T ax[2] = {(T)a.pol_ax[0], (T)a.pol_ax[1]}, ay[2] = {(T)a.pol_ay[0], (T)a.pol_ay[1]};
        const T inew = polarized_intensity<T>(Psm, BLOCK, Psm[18 * BLOCK], Psm[19 * BLOCK], Psm[20 * BLOCK], Psm[21 * BLOCK],
                                              a.pol_mode, ax, ay, status);
        r[0].i = inew;
        if (a.pol_i != nullptr) __stcs((T*)a.pol_i + base, inew);
      }
    }
    if (a.wf_opd != nullptr) {
      // OPD map against the reference sphere + exit-pupil intercepts, from the GLOBAL final state; the
      // pupil samples are re-read for the launch-plane tilt term (they were consumed by the launch)
      T wpx[RPT], wpy[RPT];
#pragma unroll
      for (int k = 0; k < RPT; ++k) { wpx[k] = 0; wpy[k] = 0; }
      if (a.px != nullptr && (a.wf.tilt[0] != 0 || a.wf.tilt[1] != 0)) {
        load_rays<T, RPT>((const T*)a.px, bin, valid, wpx);
        load_rays<T, RPT>((const T*)a.py, bin, valid, wpy);
      }
      T o0[RPT], o1[RPT], o2[RPT], o3[RPT], o4[RPT];
#pragma unroll
      for (int k = 0; k < RPT; ++k) {
        double ow, qx, qy, qz;
        wavefront_point((double)gx[k], (double)gy[k], (double)gz[k], (double)gL[k], (double)gM[k], (double)gN[k],
                        opd_value_f64(r[k]), (double)wpx[k], (double)wpy[k], a.wf, ow, qx, qy, qz);
        o0[k] = (T)ow; o1[k] = (T)qx; o2[k] = (T)qy; o3[k] = (T)qz; o4[k] = r[k].i;
      }
      store_rays<T, RPT>((T*)a.wf_opd, base, valid, o0);
      store_rays<T, RPT>((T*)a.wf_px, base, valid, o1);
      store_rays<T, RPT>((T*)a.wf_py, base, valid, o2);
      store_rays<T, RPT>((T*)a.wf_pz, base, valid, o3);
      store_rays<T, RPT>((T*)a.wf_i, base, valid, o4);
    }
    if (!(a.tflags & OLB_TF_NO_FINAL)) {
      T v[RPT];
      store_rays<T, RPT>((T*)a.x, base, valid, gx);
      store_rays<T, RPT>((T*)a.y, base, valid, gy);
      store_rays<T, RPT>((T*)a.z, base, valid, gz);
      store_rays<T, RPT>((T*)a.L, base, valid, gL);
      store_rays<T, RPT>((T*)a.M, base, valid, gM);
      store_rays<T, RPT>((T*)a.N, base, valid, gN);
#pragma unroll
      for (int k = 0; k < RPT; ++k) v[k] = r[k].i;
      store_rays<T, RPT>((T*)a.i, base, valid, v);
#pragma unroll
      for (int k = 0; k < RPT; ++k) v[k] = opd_value(r[k]);
      store_rays<T, RPT>((T*)a.opd, base, valid, v);
    }
    if constexpr ((FEAT & FEAT_POL) != 0) {
      if (a.p != nullptr) {
        using V2 = typename Vec<T, 2>::type;
        V2* dst = reinterpret_cast<V2*>((T*)a.p + base * 18);
#pragma unroll
        for (int q = 0; q < 9; ++q) {
          V2 v; v.x = Psm[(2 * q) * BLOCK]; v.y = Psm[(2 * q + 1) * BLOCK];
          __stcs(dst + q, v);
        }
      }
    }
    if constexpr ((FEAT & FEAT_EXTRA) != 0) {
      if (a.L0 != nullptr) {
        T v[RPT];
#pragma unroll
        for (int k = 0; k < RPT; ++k) v[k] = r[k].L0;
        store_rays<T, RPT>((T*)a.L0, base, valid, v);
#pragma unroll
        for (int k = 0; k < RPT; ++k) v[k] = r[k].M0;
        store_rays<T, RPT>((T*)a.M0, base, valid, v);
#pragma unroll
        for (int k = 0; k < RPT; ++k) v[k] = r[k].N0;
        store_rays<T, RPT>((T*)a.N0, base, valid, v);
      }
    }
  }
  if (status != 0 && a.status != nullptr) atomicOr(a.status, status);
  if (a.tflags & OLB_TF_MOMENTS) {
    // CTA reduction: warp tree, then one fp64 atomic per moment and warp (uniform branch: launch argument)
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      double v = mom[q];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if ((threadIdx.x & 31) == 0 && v != 0) atomicAdd(&a.moments[(size_t)sys * 8 + q], v);
    }
  }
}

// ---- backward kernel -------------------------------------------------------------------------
struct BwdArgs {
  const unsigned char* blob;
  int32_t blob_bytes;
  int32_t first, last, n_surf;
  int64_t n_rays, rec_stride, grec_stride;
  uint64_t grow_mask;    // bit r set: record row r may have a non-zero gradient (others are skipped)
  int32_t n_slots;       // per-thread gradient accumulator slots (OlbDeviceTable.bwd_slots)
  const void* in[7];     // launch state x y z L M N i
  const void* rec[8];    // forward records
  const void* grec[8];   // dLoss/d records (entries may be null)
  void* gin[8];          // dLoss/d launch state (may be null as a whole: gin[0] == null)
  double* gparams;       // n_surf * GP_COUNT, accumulated
  double* gtab;          // n_surf * GT_PER_SURFACE, accumulated: table gradients of polynomial / Zernike surfaces (or null)
};

// One ray per thread per tile.  Parameter gradients: PRIVATE fp32/fp64 accumulators per thread in
// shared memory, laid out [slot][thread] (bank-conflict free), summed over all the rays the thread
// processes in its persistent loop; reduced across the CTA once at the end (warp tree + one fp64
// global atomic per slot and CTA)  (ACC == 2).  When the table needs more slots than two resident CTAs can hold that
// way (fp64 with more than ~50 slots: configuration 3), neighbouring lanes share one accumulator after ONE shuffle
// (ACC == 1: [slot][thread / 2], half the shared memory); beyond that each surface's contributions are
// warp-reduced immediately (ACC == 0: five shuffles per value).  Both precisions ask for 2 resident CTAs per SM.
// POLY: the table holds polynomial / Zernike surfaces (table gradients wanted); false compiles those paths out.
template <typename T, int ACC, bool POLY>
__global__ void __launch_bounds__(BLOCK, 2) trace_bwd_kernel(const __grid_constant__ BwdArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem);
  unsigned char* tab = smem + 16;
  stage_table(tab, a.blob, (uint32_t)a.blob_bytes, bar);
  const PrepHeader* H = reinterpret_cast<const PrepHeader*>(tab);
  const PrepSurface<T>* surf = reinterpret_cast<const PrepSurface<T>*>(tab + sizeof(PrepHeader));
  const T* pool = reinterpret_cast<const T*>(surf + H->n_surf);
  unsigned char* after = tab + ((a.blob_bytes + 15) & ~15);
  constexpr bool SMEM_ACC = ACC == 2;                    // one accumulator column per thread
  constexpr bool PAIR_ACC = ACC == 1;                    // ... per pair of neighbouring lanes
  constexpr int ACC_COLS = SMEM_ACC ? BLOCK : BLOCK / 2;
  T* tacc = reinterpret_cast<T*>(after);                 // ACC 2 / 1: [n_slots][ACC_COLS]
  double* wacc = reinterpret_cast<double*>(after);       // ACC 0: [n_surf * GP_COUNT]
  const int n_slots = a.n_slots;
  if (ACC != 0) {
    for (int q = threadIdx.x; q < n_slots * ACC_COLS; q += BLOCK) tacc[q] = 0;
  } else {
    for (int q = threadIdx.x; q < a.n_surf * GP_COUNT; q += BLOCK) wacc[q] = 0.0;
  }
  __syncthreads();

  const int64_t n = a.n_rays;
  const int64_t n_tiles = (n + BLOCK - 1) / BLOCK;
  const int lane = threadIdx.x & 31;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t k = tile * BLOCK + threadIdx.x;
    const bool valid = k < n;
    if (SMEM_ACC && !POLY && !valid) continue;    // (warp reductions need the whole warp)
    const int64_t kk = valid ? k : 0;
    Adjoint<T> ad{0, 0, 0, 0, 0, 0, 0, 0};
    // Software-pipelined walk from the image surface back to the first one.  Surface s needs the state
    // BEFORE it (record row s-1, or the launch state for s == first), the intercept AFTER it (row s: x y z)
    // and dLoss/d(row s).  Row s-1 is fetched while surface s is being differentiated, and its x y z are
    // reused as the "after" intercept of surface s-1, so every record value is loaded exactly once and the
    // load latency overlaps the arithmetic of the previous surface (long_scoreboard was the top stall).
    T pre[7] = {0, 0, 0, 0, 0, 0, 0}, post[3] = {0, 0, 0}, g8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    auto load_state = [&](int s, T* dst) {             // state in front of surface s
      if (s == a.first) {
#pragma unroll
        for (int q = 0; q < 7; ++q) dst[q] = __ldcs((const T*)a.in[q] + kk);
      } else {
        const int64_t off = (int64_t)(s - 1 - a.first) * a.rec_stride + kk;
#pragma unroll
        for (int q = 0; q < 7; ++q) dst[q] = __ldcs((const T*)a.rec[q] + off);
      }
    };
    auto load_grad = [&](int s, T* dst) {              // dLoss/d(record row of surface s)
#pragma unroll
      for (int q = 0; q < 8; ++q) dst[q] = 0;
      if ((a.grow_mask >> (s - a.first)) & 1ull) {
        const int64_t goff = (int64_t)(s - a.first) * a.grec_stride + kk;
#pragma unroll
        for (int q = 0; q < 8; ++q)
          if (a.grec[q]) dst[q] = __ldcs((const T*)a.grec[q] + goff);
      }
    };
    // fp64 keeps the loads at the top of each iteration: the second register set of the pipeline costs it
    // the second resident CTA (160 registers; measured 4.9 ms vs 3.3 ms), fp32 gains 29 % from it.
    constexpr bool PIPE = sizeof(T) == 4;
    if (valid) {
      const int sl = a.last - 1;
      const int64_t off = (int64_t)(sl - a.first) * a.rec_stride + kk;
      post[0] = __ldcs((const T*)a.rec[0] + off); post[1] = __ldcs((const T*)a.rec[1] + off);
      post[2] = __ldcs((const T*)a.rec[2] + off);
      if (PIPE) {
        load_grad(sl, g8);
        load_state(sl, pre);
      }
    }
    for (int s = a.last - 1; s >= a.first; --s) {
      const PrepSurface<T>& S = surf[s];
      const bool noop = S.kind == OLB_GEOM_NOOP;
      if (!PIPE && valid) {
        load_grad(s, g8);
        load_state(s, pre);
      }
      T pren[7] = {0, 0, 0, 0, 0, 0, 0}, g8n[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (PIPE && valid && s > a.first) {              // prefetch for surface s-1
        load_grad(s - 1, g8n);
        load_state(s - 1, pren);
      }
      ad.x += g8[0]; ad.y += g8[1]; ad.z += g8[2]; ad.L += g8[3]; ad.M += g8[4]; ad.N += g8[5]; ad.i += g8[6]; ad.opd += g8[7];
      PolyAdj<T> pa;
      pa.active = 0;
      if (!noop) {   // (a NOOP surface records its input unchanged: the adjoint passes through)
        T pg[GP_SCALARS];
#pragma unroll
        for (int q = 0; q < GP_SCALARS; ++q) pg[q] = 0;
        // slots of this surface: 7 scalars, its even-asphere coefficients, then dLoss/dR (9) if the pose is tilted
        const int ncoef = coef_grad_slots(S);
        const bool tilted = (S.flags & OLB_SF_ROTATED) != 0;
        if (SMEM_ACC) {
          T* mine = tacc + (int64_t)S.gslot * BLOCK + threadIdx.x;
          if (valid)
            surface_backward<T, POLY>(S, pool, pre[0], pre[1], pre[2], pre[3], pre[4], pre[5], pre[6], post[0], post[1], post[2],
                                      ad, pg, tilted ? mine + (GP_COEF + ncoef) * BLOCK : nullptr, BLOCK, POLY ? &pa : nullptr);
          // pose, curvature, conic, n1, n2: every surface has these 7; only even aspheres have more
#pragma unroll
          for (int q = 0; q < GP_COEF; ++q) mine[q * BLOCK] += pg[q];
          if (ncoef > 0) {
#pragma unroll
            for (int q = GP_COEF; q < GP_SCALARS; ++q)
              if (q < GP_COEF + ncoef) mine[q * BLOCK] += pg[q];
          }
        } else if (PAIR_ACC) {
          T r9[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
          if (valid)
            surface_backward<T, POLY>(S, pool, pre[0], pre[1], pre[2], pre[3], pre[4], pre[5], pre[6], post[0], post[1], post[2],
                                      ad, pg, tilted ? r9 : nullptr, 1, POLY ? &pa : nullptr);
          // lanes 2k and 2k+1 share column k: one shuffle, the even lane accumulates
          T* mine = tacc + (int64_t)S.gslot * ACC_COLS + (threadIdx.x >> 1);
          const bool even = (lane & 1) == 0;
#pragma unroll
          for (int q = 0; q < GP_SCALARS; ++q) {
            if (q >= GP_COEF + ncoef) break;
            const T v = pg[q] + __shfl_xor_sync(0xffffffffu, pg[q], 1);
            if (even) mine[q * ACC_COLS] += v;
          }
          if (tilted) {
#pragma unroll
            for (int q = 0; q < 9; ++q) {
              const T v = r9[q] + __shfl_xor_sync(0xffffffffu, r9[q], 1);
              if (even) mine[(GP_COEF + ncoef + q) * ACC_COLS] += v;
            }
          }
        } else {
          T r9[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
          if (valid)
            surface_backward<T, POLY>(S, pool, pre[0], pre[1], pre[2], pre[3], pre[4], pre[5], pre[6], post[0], post[1], post[2],
                                      ad, pg, tilted ? r9 : nullptr, 1, POLY ? &pa : nullptr);
#pragma unroll
          for (int q = 0; q < GP_SCALARS; ++q) {
            if (q >= GP_COEF + ncoef) break;
            T v = pg[q];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0 && v != 0) atomicAdd(&wacc[s * GP_COUNT + q], (double)v);
          }
          if (tilted) {
#pragma unroll
            for (int q = 0; q < 9; ++q) {
              T v = r9[q];
#pragma unroll
              for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
              if (lane == 0 && v != 0) atomicAdd(&wacc[s * GP_COUNT + GP_R + q], (double)v);
            }
          }
        }
      }
      if (POLY && a.gtab != nullptr && poly_family_kind(S.kind)) {
        // Table gradients of a polynomial-family surface (warp-uniform branch; every lane takes part in the
        // reductions, inactive rays contribute zeros): dLoss/dS_ij += q xn^i yn^j, dLoss/dD_ij += ax i xn^(i-1) yn^j +
        // ay j xn^i yn^(j-1); one fp64 atomic per entry and warp.
        double* gS = a.gtab + (size_t)s * GT_PER_SURFACE;
        double* gD = gS + GT_BLOCK;
        const bool tri = (S.flags & PSF_POLY_TRI) != 0;
        const bool on = pa.active != 0;
        T xi = 1, xim = 0;
        for (int i = 0; i < S.poly_rows; ++i) {
          T yj = 1, yjm = 0;
          const int jmax = tri ? (S.poly_rows - 1 - i) : (S.poly_cols - 1);
          for (int j = 0; j <= jmax; ++j) {
            T vS = 0, vD = 0;
            if (on) poly_table_terms(pa, i, j, xi, xim, yj, yjm, vS, vD);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
              vS += __shfl_xor_sync(0xffffffffu, vS, o);
              vD += __shfl_xor_sync(0xffffffffu, vD, o);
            }
            if (lane == 0) {
              if (vS != 0) atomicAdd(&gS[i * GT_DIM + j], (double)vS);
              if (vD != 0) atomicAdd(&gD[i * GT_DIM + j], (double)vD);
            }
            if (on) { yjm = yj; yj *= pa.yn; }
          }
          if (on) { xim = xi; xi *= pa.xn; }
        }
      }
      post[0] = pre[0]; post[1] = pre[1]; post[2] = pre[2];
      if (PIPE) {
#pragma unroll
        for (int q = 0; q < 7; ++q) pre[q] = pren[q];
#pragma unroll
        for (int q = 0; q < 8; ++q) g8[q] = g8n[q];
      }
    }
    if (valid && a.gin[0]) {
      __stcs((T*)a.gin[0] + k, ad.x); __stcs((T*)a.gin[1] + k, ad.y); __stcs((T*)a.gin[2] + k, ad.z);
      __stcs((T*)a.gin[3] + k, ad.L); __stcs((T*)a.gin[4] + k, ad.M); __stcs((T*)a.gin[5] + k, ad.N);
      __stcs((T*)a.gin[6] + k, ad.i); __stcs((T*)a.gin[7] + k, ad.opd);
    }
  }
  __syncthreads();
  if (ACC != 0) {
    // CTA reduction: warp w sums slots w, w+8, ...: 8 (4) values per lane, tree, one fp64 atomic
    const int warp = threadIdx.x >> 5;
    for (int s = 0; s < a.n_surf; ++s) {
      const PrepSurface<T>& S = surf[s];
      for (int q = warp; q < S.gslots; q += BLOCK / 32) {
        const T* col = tacc + (int64_t)(S.gslot + q) * ACC_COLS;
        double v = 0;
        for (int j = lane; j < ACC_COLS; j += 32) v += (double)col[j];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        // slot -> parameter: scalars and coefficients in place, the tilted pose's 9 slots -> GP_R ..
        const int ncoef = coef_grad_slots(S);
        const int qp = q < GP_COEF + ncoef ? q : GP_R + (q - GP_COEF - ncoef);
        if (lane == 0 && v != 0) atomicAdd(&a.gparams[s * GP_COUNT + qp], v);
      }
    }
  } else {
    for (int q = threadIdx.x; q < a.n_surf * GP_COUNT; q += BLOCK)
      if (wacc[q] != 0.0) atomicAdd(&a.gparams[q], wacc[q]);
  }
}

template <typename T>
static int trace_bwd_impl(const OlbDeviceTable* wh, int32_t first, int32_t last, const OlbRays* rays_in,
                          const OlbRecords* rec, const OlbRecords* grec, const OlbRays* gin, double* gparams,
                          double* gtab, int64_t n_rays, uint64_t grow_mask, cudaStream_t stream) {
  if (!wh || wh->magic != WS_MAGIC || !wh->workspace)
    return fail(OLB_ERR_INVALID_ARG, "table handle was not initialised by olb_table_upload");
  if (!wh->bwd_supported)
    return fail(OLB_ERR_UNSUPPORTED, "backward: table not supported (a geometry other than plane / standard / even- and "
                                     "odd-asphere / polynomial / Zernike, a Fresnel coating or several wavelengths)");
  if (wh->bwd_supported == 2 && !gtab)
    return fail(OLB_ERR_UNSUPPORTED, "backward: the table has polynomial / Zernike surfaces: grad_tables is required");
  if (!rays_in || !rec || !gparams) return fail(OLB_ERR_INVALID_ARG, "rays_in, rec and grad_params are required");
  if (first < 0 || last > wh->n_surfaces || first > last) return fail(OLB_ERR_INVALID_ARG, "bad surface range");
  if (n_rays <= 0 || first == last) return OLB_OK;
  BwdArgs a{};
  a.blob = (const unsigned char*)wh->workspace + (sizeof(T) == 8 ? wh->off_f64 : wh->off_f32);
  a.blob_bytes = sizeof(T) == 8 ? wh->bytes_f64 : wh->bytes_f32;
  a.first = first; a.last = last; a.n_surf = wh->n_surfaces; a.n_rays = n_rays;
  const void* in[7] = {rays_in->x, rays_in->y, rays_in->z, rays_in->L, rays_in->M, rays_in->N, rays_in->i};
  const void* rr[8] = {rec->x, rec->y, rec->z, rec->L, rec->M, rec->N, rec->intensity, rec->opd};
  for (int q = 0; q < 7; ++q) { if (!in[q]) return fail(OLB_ERR_INVALID_ARG, "a launch-state array is NULL"); a.in[q] = in[q]; }
  for (int q = 0; q < 8; ++q) { if (!rr[q]) return fail(OLB_ERR_INVALID_ARG, "backward needs all 8 record arrays"); a.rec[q] = rr[q]; }
  a.rec_stride = rec->row_stride;
  if (a.rec_stride < n_rays) return fail(OLB_ERR_INVALID_ARG, "record row_stride < n_rays");
  if (grec) {
    const void* gg[8] = {grec->x, grec->y, grec->z, grec->L, grec->M, grec->N, grec->intensity, grec->opd};
    for (int q = 0; q < 8; ++q) a.grec[q] = gg[q];
    a.grec_stride = grec->row_stride;
    if (a.grec_stride < n_rays) return fail(OLB_ERR_INVALID_ARG, "grad record row_stride < n_rays");
  }
  if (gin) {
    void* go[8] = {gin->x, gin->y, gin->z, gin->L, gin->M, gin->N, gin->i, gin->opd};
    for (int q = 0; q < 8; ++q) { if (!go[q]) return fail(OLB_ERR_INVALID_ARG, "grad_rays_in needs all 8 arrays"); a.gin[q] = go[q]; }
  }
  a.gparams = gparams;
  a.gtab = wh->bwd_supported == 2 ? gtab : nullptr;
  a.grow_mask = grow_mask;
  a.n_slots = wh->bwd_slots;
  const size_t base_smem = 16 + (((size_t)a.blob_bytes + 15) & ~size_t(15));
  const size_t smem_acc = base_smem + (size_t)wh->bwd_slots * BLOCK * sizeof(T);
  const size_t smem_warp = base_smem + (size_t)wh->n_surfaces * GP_COUNT * sizeof(double);
  const size_t smem_pair = base_smem + (size_t)wh->bwd_slots * (BLOCK / 2) * sizeof(T);
  // 2 CTAs per SM must still fit: 228 KB per SM, 1 KB of it reserved per resident CTA -> 113 KB each
  const int acc = smem_acc <= 113 * 1024 ? 2 : (smem_pair <= 113 * 1024 ? 1 : 0);
  const bool poly = a.gtab != nullptr;
  auto kern = acc == 2 ? (poly ? trace_bwd_kernel<T, 2, true> : trace_bwd_kernel<T, 2, false>)
            : acc == 1 ? (poly ? trace_bwd_kernel<T, 1, true> : trace_bwd_kernel<T, 1, false>)
                       : (poly ? trace_bwd_kernel<T, 0, true> : trace_bwd_kernel<T, 0, false>);
  const size_t smem = acc == 2 ? smem_acc : acc == 1 ? smem_pair : smem_warp;
  if (smem > 48 * 1024) OLB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int dev = 0, num_sms = 0, per_sm = 0;
  OLB_CUDA(cudaGetDevice(&dev));
  OLB_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
  OLB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, BLOCK, smem));
  if (per_sm < 1) return fail(OLB_ERR_CUDA, "backward kernel does not fit on an SM");
  // the backward pass is read-dominated: one resident wave is best (measured 1.52 ms vs 1.84 ms at 64x)
  int64_t grid = (int64_t)num_sms * per_sm;
  const int64_t n_tiles = (n_rays + BLOCK - 1) / BLOCK;
  if (grid > n_tiles) grid = n_tiles;
  kern<<<(unsigned)grid, BLOCK, smem, stream>>>(a);
  OLB_CUDA(cudaGetLastError());
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return OLB_OK;
}

// ---- launcher -------------------------------------------------------------------------------
template <typename T, int RPT, uint32_t FEAT>
static int launch_instance(const TraceArgs& a, cudaStream_t stream) {
  auto kern = trace_kernel<T, RPT, FEAT>;
  const size_t smem = (FEAT & FEAT_POL) ? 16 + (((size_t)a.blob_bytes + 15) & ~size_t(15)) + (size_t)POL_SLOTS * BLOCK * sizeof(T)
                                        : 16 + (size_t)a.blob_bytes;
  static thread_local int cached_dev = -1;
  static thread_local int num_sms = 0;
  static thread_local int blocks_per_sm = 0;
  static thread_local size_t cached_smem = 0;
  int dev = 0;
  OLB_CUDA(cudaGetDevice(&dev));
  if (dev != cached_dev || smem != cached_smem) {
    if (smem > 48 * 1024) {
      OLB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    OLB_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
    OLB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, kern, BLOCK, smem));
    if (blocks_per_sm < 1) return fail(OLB_ERR_CUDA, "kernel does not fit on an SM (table too large?)");
    cached_dev = dev;
    cached_smem = smem;
  }
  const int64_t per_tile = (int64_t)BLOCK * RPT;
  if (a.sys_rays > 0) {
    // batched systems: grid.y = system, grid.x = tiles of one system (one tile per CTA, grid-stride beyond 65535)
    const int64_t n_sys = a.n_rays / a.sys_rays;
    int64_t gx = (a.sys_rays + per_tile - 1) / per_tile;
    if (gx > 65535) gx = 65535;
    if (n_sys > 65535) return fail(OLB_ERR_INVALID_ARG, "more than 65535 systems in one batch");
    kern<<<dim3((unsigned)gx, (unsigned)n_sys), BLOCK, smem, stream>>>(a);
    OLB_CUDA(cudaGetLastError());
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return OLB_OK;
  }
  const int64_t n_tiles = (a.n_rays + per_tile - 1) / per_tile;
  // Grid: OVER-SUBSCRIBED grid-stride loop, 64 x the resident CTA count (capped at one tile per CTA).
  // A one-wave persistent grid keeps all CTAs in lock-step (everybody loads, then everybody stores row
  // r ...); staggered CTA start times spread the concurrent write streams.  On an H100 (Double-Gauss,
  // 10 M rays, full records) 64x and 16x tie, 4x and 1x are 3-4 % slower in fp32.
  int64_t grid = (int64_t)num_sms * blocks_per_sm * 64;
  if (grid > n_tiles) grid = n_tiles;
  if (grid < 1) return OLB_OK;
  kern<<<(unsigned)grid, BLOCK, smem, stream>>>(a);
  OLB_CUDA(cudaGetLastError());
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return OLB_OK;
}

constexpr uint32_t FEAT_GENERAL = FEAT_ROT | FEAT_NEWTON | FEAT_EXTRA | FEAT_FREEFORM;
// What a Q-2D table may not hold: its two kernel variants carry none of these code paths
constexpr uint32_t FEAT_Q2D_EXCLUDED = FEAT_PHASE | FEAT_GRATING | FEAT_GRID | FEAT_POLYGON | FEAT_BSDF | FEAT_JONES;
static const char* const Q2D_EXCLUDED_MSG = "a Forbes Q-2D surface in a table with a phase profile, ruled grating, grid "
                                            "sag, polygon aperture, BSDF or thin-film / polarizer / retarder coating is not built";

template <typename T, int RPT>
static int launch_feat(const TraceArgs& a, uint32_t features, cudaStream_t stream) {
  if (features & FEAT_POL) {
    if constexpr (RPT == 1) {
      // lean polarized variants for the common systems: the general kernel's code does not fit the instruction
      // cache (no_instruction was the second largest stall of the Zernike + Fresnel configuration)
      const uint32_t g = features & ~FEAT_POL;
      if (g & FEAT_BSDF) return fail(OLB_ERR_UNSUPPORTED, "polarized trace of a table with a BSDF surface is not built");
      if (g & FEAT_Q2D) {      // Forbes Q-2D surfaces: the general polarized kernel + the Q-2D sag, and nothing else
        if (g & FEAT_Q2D_EXCLUDED) return fail(OLB_ERR_UNSUPPORTED, Q2D_EXCLUDED_MSG);
        return launch_instance<T, 1, FEAT_GENERAL | FEAT_POL | FEAT_Q2D>(a, stream);
      }
      if (g & FEAT_POLYGON)      // polygon apertures: the grid-sag superset + the polygon scan, so a polygon works on any surface
        return launch_instance<T, 1, FEAT_GENERAL | FEAT_PHASE | FEAT_GRATING | FEAT_POL | FEAT_JONES | FEAT_GRID | FEAT_POLYGON>(a, stream);
      if (g & FEAT_GRID)         // grid-sag surfaces: the superset below, so every coating and DOE works on a grid
        return launch_instance<T, 1, FEAT_GENERAL | FEAT_PHASE | FEAT_GRATING | FEAT_POL | FEAT_JONES | FEAT_GRID>(a, stream);
      if (g & FEAT_JONES)        // thin-film / polarizer / retarder coatings, on any surface (DOEs and gratings too)
        return launch_instance<T, 1, FEAT_GENERAL | FEAT_PHASE | FEAT_GRATING | FEAT_POL | FEAT_JONES>(a, stream);
      if (g & FEAT_GRATING)                                                                            // gratings (+ phase)
        return launch_instance<T, 1, FEAT_GENERAL | FEAT_PHASE | FEAT_GRATING | FEAT_POL>(a, stream);
      if (g & FEAT_PHASE) return launch_instance<T, 1, FEAT_GENERAL | FEAT_PHASE | FEAT_POL>(a, stream);  // phase profiles
      if (g == 0) return launch_instance<T, 1, FEAT_POL>(a, stream);                                   // planes / conics
      if ((g & ~(FEAT_NEWTON | FEAT_FREEFORM)) == 0)
        return launch_instance<T, 1, FEAT_NEWTON | FEAT_FREEFORM | FEAT_POL>(a, stream);               // + Newton families
      return launch_instance<T, 1, FEAT_GENERAL | FEAT_POL>(a, stream);
    } else {
      return fail(OLB_ERR_UNSUPPORTED, "polarized trace uses one ray per thread");
    }
  }
  // phase-profile tables: the general kernel plus the phase interaction, one ray per thread for either caller RPT;
  // tables with a ruled grating (phase surfaces allowed beside it) add the grating interaction to that, and tables with
  // a grid-sag surface the grid loop to both; tables with a polygon aperture the polygon scan to all three; tables with
  // a BSDF surface the scatter to all four, so a BSDF works on every geometry, interaction and aperture
  if (features & FEAT_Q2D) {    // Forbes Q-2D surfaces: the general kernel + the Q-2D sag, one ray per thread
    if (features & FEAT_Q2D_EXCLUDED) return fail(OLB_ERR_UNSUPPORTED, Q2D_EXCLUDED_MSG);
    return launch_instance<T, 1, FEAT_GENERAL | FEAT_Q2D>(a, stream);
  }
  if (features & FEAT_BSDF)
    return launch_instance<T, 1, FEAT_GENERAL | FEAT_PHASE | FEAT_GRATING | FEAT_GRID | FEAT_POLYGON | FEAT_BSDF>(a, stream);
  if (features & FEAT_POLYGON)
    return launch_instance<T, 1, FEAT_GENERAL | FEAT_PHASE | FEAT_GRATING | FEAT_GRID | FEAT_POLYGON>(a, stream);
  if (features & FEAT_GRID) return launch_instance<T, 1, FEAT_GENERAL | FEAT_PHASE | FEAT_GRATING | FEAT_GRID>(a, stream);
  if (features & FEAT_GRATING) return launch_instance<T, 1, FEAT_GENERAL | FEAT_PHASE | FEAT_GRATING>(a, stream);
  if (features & FEAT_PHASE) return launch_instance<T, 1, FEAT_GENERAL | FEAT_PHASE>(a, stream);
  if (features == 0) return launch_instance<T, RPT, 0u>(a, stream);
  if (features == FEAT_ROT) return launch_instance<T, RPT, FEAT_ROT>(a, stream);
  if (features == FEAT_NEWTON) return launch_instance<T, RPT, FEAT_NEWTON>(a, stream);                        // aspheres
  if (features == (FEAT_NEWTON | FEAT_FREEFORM)) return launch_instance<T, RPT, FEAT_NEWTON | FEAT_FREEFORM>(a, stream);
  return launch_instance<T, RPT, FEAT_GENERAL>(a, stream);
}

// fp32 x 4 rays/thread exists only for the closed-form feature sets (code size, registers).
template <typename T, int RPT>
static int launch_feat_cf(const TraceArgs& a, uint32_t features, cudaStream_t stream) {
  if (features & FEAT_POL) return fail(OLB_ERR_UNSUPPORTED, "polarized tables run one ray per thread (internal dispatch error)");
  if (features == 0) return launch_instance<T, RPT, 0u>(a, stream);
  return launch_instance<T, RPT, FEAT_ROT>(a, stream);
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

template <typename T>
static int trace_impl(const OlbDeviceTable* wh, const OlbTraceCall& c, cudaStream_t stream, int64_t ray0 = 0) {
  if (!wh || wh->magic != WS_MAGIC || !wh->workspace)
    return fail(OLB_ERR_INVALID_ARG, "table handle was not initialised by olb_table_upload");
  const unsigned char* workspace_dev = (const unsigned char*)wh->workspace;
  const int32_t first = c.first, last = c.last;
  const int64_t n_rays = c.n_rays, rays_per_system = c.rays_per_system;
  uint32_t flags = c.flags;
  const OlbPupilLaunch* launch = c.launch;
  double* moments = c.moments;
  const OlbWavefrontRef* wref = c.wavefront_ref;
  const OlbWavefrontOut* wout = c.wavefront_out;
  const OlbPolarization* pol = c.pol;
  const OlbRecords* rec = c.rec;
  const OlbRays none{};
  const OlbRays* rays = c.rays ? c.rays : &none;   // pupil launch / NO_FINAL: the ray arrays may all be NULL
  if (n_rays < 0) return fail(OLB_ERR_INVALID_ARG, "n_rays < 0");
  if (rays_per_system < 0) return fail(OLB_ERR_INVALID_ARG, "rays_per_system < 0");
  if (first < 0 || last > wh->n_surfaces || first > last) return fail(OLB_ERR_INVALID_ARG, "bad surface range");
  if (wh->n_systems > 1 && rays_per_system == 0)
    return fail(OLB_ERR_INVALID_ARG, "this table holds several systems: set rays_per_system");
  if (n_rays == 0 || first == last) return OLB_OK;
  void* req[] = {rays->x, rays->y, rays->z, rays->L, rays->M, rays->N, rays->i, rays->opd};
  if (moments) flags |= OLB_TF_MOMENTS; else flags &= ~uint32_t(OLB_TF_MOMENTS);
  const bool need_state = launch == nullptr || !(flags & OLB_TF_NO_FINAL);
  for (void* p : req) {
    if (!p && need_state) return fail(OLB_ERR_INVALID_ARG, "a required ray array is NULL");
    if (p && !aligned16(p)) return fail(OLB_ERR_ALIGNMENT, "ray array not 16-byte aligned");
  }
  if (launch) {
    if (!launch->Px || !launch->Py) return fail(OLB_ERR_INVALID_ARG, "launch.Px / launch.Py is NULL");
    if (!aligned16(launch->Px) || !aligned16(launch->Py)) return fail(OLB_ERR_ALIGNMENT, "launch.Px / Py not 16-byte aligned");
    if (flags & OLB_TF_POLARIZED) flags |= OLB_TF_POL_IDENTITY;   // PolarizedRays.__init__: P starts as the identity
  }
  if (wh->n_wl > 1) {
    if (!rays->w) return fail(OLB_ERR_INVALID_ARG, "rays.w is NULL but the table has several wavelengths");
    if (!aligned16(rays->w)) return fail(OLB_ERR_ALIGNMENT, "rays.w not 16-byte aligned");
  }
  TraceArgs a{};
  a.blob = workspace_dev + (sizeof(T) == 8 ? wh->off_f64 : wh->off_f32);
  a.blob_bytes = sizeof(T) == 8 ? wh->bytes_f64 : wh->bytes_f32;
  a.first = first; a.last = last; a.tflags = flags; a.n_rays = n_rays;
  a.x = rays->x; a.y = rays->y; a.z = rays->z; a.L = rays->L; a.M = rays->M; a.N = rays->N;
  a.i = rays->i; a.w = rays->w; a.opd = rays->opd;
  a.L0 = rays->L0; a.M0 = rays->M0; a.N0 = rays->N0; a.p = rays->p;
  a.status = c.status;
  a.tflags = flags;
  a.ray0 = ray0;
  a.rng_stream = c.rng_stream;
  if (rays_per_system > 0) {
    if (wh->n_systems < 1 || n_rays != rays_per_system * (int64_t)wh->n_systems)
      return fail(OLB_ERR_INVALID_ARG, "batched trace: n_rays must equal rays_per_system * n_systems of the table");
    if (flags & OLB_TF_POLARIZED) return fail(OLB_ERR_UNSUPPORTED, "batched trace with polarized rays is not built");
    a.sys_rays = rays_per_system;
    a.blob_stride = sizeof(T) == 8 ? wh->stride_f64 : wh->stride_f32;
    a.shared_in = (flags & OLB_TF_SHARED_INPUT) ? 1 : 0;
    if (a.shared_in && !(flags & OLB_TF_NO_FINAL))
      return fail(OLB_ERR_INVALID_ARG, "OLB_TF_SHARED_INPUT needs OLB_TF_NO_FINAL (results go to records / moments)");
  }
  if (moments) { a.moments = moments; a.mcx = c.center[0]; a.mcy = c.center[1]; }
  if (wref || wout) {
    if (!wref || !wout) return fail(OLB_ERR_INVALID_ARG, "wavefront: ref and out are both required");
    void* wo[] = {wout->opd, wout->pupil_x, wout->pupil_y, wout->pupil_z, wout->intensity};
    for (void* p : wo) {
      if (!p) return fail(OLB_ERR_INVALID_ARG, "wavefront: an output array is NULL");
      if (!aligned16(p)) return fail(OLB_ERR_ALIGNMENT, "wavefront output array not 16-byte aligned");
    }
    if (!(wref->radius > 0) || !(wref->n_image > 0) || !(wref->wavelength_um > 0))
      return fail(OLB_ERR_INVALID_ARG, "wavefront: radius, n_image and wavelength must be positive");
    if ((wref->tilt[0] != 0 || wref->tilt[1] != 0) && !launch)
      return fail(OLB_ERR_INVALID_ARG, "wavefront: the launch-plane tilt term needs the pupil samples (launch)");
    if (rays_per_system > 0)
      return fail(OLB_ERR_UNSUPPORTED, "wavefront epilogue with batched systems is not built");
    if (last != wh->n_surfaces) return fail(OLB_ERR_INVALID_ARG, "wavefront: the trace must end on the image surface");
    a.wf_opd = wout->opd; a.wf_px = wout->pupil_x; a.wf_py = wout->pupil_y; a.wf_pz = wout->pupil_z; a.wf_i = wout->intensity;
    for (int q = 0; q < 3; ++q) a.wf.c[q] = wref->center[q];
    a.wf.R = wref->radius; a.wf.n_image = wref->n_image; a.wf.tilt[0] = wref->tilt[0]; a.wf.tilt[1] = wref->tilt[1];
    a.wf.opd_ref = wref->opd_ref; a.wf.inv_wl = 1.0 / (wref->wavelength_um * 1e-3);
  }
  if (launch) {
    a.px = launch->Px; a.py = launch->Py;
    for (int q = 0; q < 3; ++q) { a.lo0[q] = launch->origin0[q]; a.lt0[q] = launch->target0[q]; }
    for (int q = 0; q < 2; ++q) { a.los[q] = launch->origin_scale[q]; a.lts[q] = launch->target_scale[q]; }
    a.linten = launch->intensity;
    if (launch->Hx || launch->Hy) {
      if (!launch->Hx || !launch->Hy) return fail(OLB_ERR_INVALID_ARG, "launch.Hx and launch.Hy go together");
      if (!aligned16(launch->Hx) || !aligned16(launch->Hy)) return fail(OLB_ERR_ALIGNMENT, "launch.Hx / Hy not 16-byte aligned");
      if (launch->field_mode != 1 && launch->field_mode != 2) return fail(OLB_ERR_INVALID_ARG, "launch.field_mode must be 1 (angle) or 2 (object height)");
      a.hx = launch->Hx; a.hy = launch->Hy; a.fmode = launch->field_mode; a.farg = launch->field_arg;
      for (int q = 0; q < 2; ++q) { a.lof[q] = launch->origin_field[q]; a.ltf[q] = launch->target_field[q]; }
      if (launch->n_vig < 0 || launch->n_vig > OLB_MAX_VIG_FIELDS) return fail(OLB_ERR_INVALID_ARG, "launch.n_vig out of range");
      if (launch->n_vig > 0 && (launch->vig_power < 1 || launch->vig_power > 2)) return fail(OLB_ERR_INVALID_ARG, "launch.vig_power must be 1 or 2");
      a.n_vig = launch->n_vig; a.vig_power = launch->vig_power;
      for (int j = 0; j < launch->n_vig; ++j)
        for (int q = 0; q < 4; ++q) a.vig[j][q] = launch->vig[j][q];
    }
  }
  uint32_t features = wh->features;
  if (flags & OLB_TF_POLARIZED) features |= FEAT_POL;
  if (pol) {
    if (!(flags & OLB_TF_POLARIZED)) return fail(OLB_ERR_INVALID_ARG, "polarization epilogue needs OLB_TF_POLARIZED");
    if (pol->intensity && !aligned16(pol->intensity)) return fail(OLB_ERR_ALIGNMENT, "pol.intensity not 16-byte aligned");
    if ((flags & OLB_TF_NO_FINAL) && !pol->intensity && !wout)
      return fail(OLB_ERR_INVALID_ARG, "polarization epilogue with OLB_TF_NO_FINAL needs pol.intensity (or the wavefront outputs)");
    a.pol_mode = pol->is_polarized ? 1 : 2;
    a.pol_ax[0] = pol->Ex * cos(pol->phase_x); a.pol_ax[1] = pol->Ex * sin(pol->phase_x);
    a.pol_ay[0] = pol->Ey * cos(pol->phase_y); a.pol_ay[1] = pol->Ey * sin(pol->phase_y);
    a.pol_i = pol->intensity;
  }
  if (rays->L0 || rays->M0 || rays->N0) {
    if (!(rays->L0 && rays->M0 && rays->N0)) return fail(OLB_ERR_INVALID_ARG, "L0/M0/N0 must be all set or all NULL");
    if (!aligned16(rays->L0) || !aligned16(rays->M0) || !aligned16(rays->N0))
      return fail(OLB_ERR_ALIGNMENT, "L0/M0/N0 not 16-byte aligned");
    features |= FEAT_EXTRA;
  }
  constexpr int V = sizeof(T) == 4 ? 4 : 2;
  bool vec_ok = true, rec_stride_ok2 = true;
  if (rays_per_system > 0) {   // every system's segment must start on a vector boundary
    if (rays_per_system % V) vec_ok = false;
    if (rays_per_system % 2) rec_stride_ok2 = false;
  }
  if (rec) {
    void* rr[] = {rec->x, rec->y, rec->z, rec->L, rec->M, rec->N, rec->intensity, rec->opd};
    int n_set = 0;
    for (void* p : rr) n_set += p != nullptr;
    if (n_set != 0 && n_set != 8)
      return fail(OLB_ERR_INVALID_ARG, "record arrays must be all set or all NULL");
    if (n_set == 8) {
      for (void* p : rr)
        if (!aligned16(p)) return fail(OLB_ERR_ALIGNMENT, "record array not 16-byte aligned");
      if (rec->row_stride < n_rays) return fail(OLB_ERR_INVALID_ARG, "record row_stride < n_rays");
      a.rx = rec->x; a.ry = rec->y; a.rz = rec->z; a.rL = rec->L; a.rM = rec->M; a.rN = rec->N;
      a.ri = rec->intensity; a.ropd = rec->opd; a.rec_stride = rec->row_stride;
      if (rec->row_stride % V) vec_ok = false;
      if (rec->row_stride % 2) rec_stride_ok2 = false;
    }
  }
  if ((flags & OLB_TF_NO_FINAL) && !a.rx && !moments && !a.wf_opd)
    return fail(OLB_ERR_INVALID_ARG, "OLB_TF_NO_FINAL needs record arrays, moments or wavefront outputs (the result would be lost)");
  // Rays per thread.  Closed-form tables (planes / conics, optionally rotated): fp32 -> 4
  // (float4 accesses), fp64 -> 2 (double2 accesses; on an H100 the Double-Gauss at 10 M rays with full
  // records traces in 3.25 ms against 3.33 ms with one ray per thread).  Tables with
  // Newton surfaces / aperture programs / coatings: fp32 -> 2, fp64 -> 1 (their per-ray code
  // is large; more rays per thread only spills).
  if (features & FEAT_POL) {
    if (!(flags & OLB_TF_POLARIZED))
      return fail(OLB_ERR_INVALID_ARG, "table has Fresnel coatings: needs OLB_TF_POLARIZED and rays.p "
                                       "(the reference raises for polarization == 'ignore', ray_generator.py:90-94)");
    // rays.p may be omitted only when nothing would be lost: P starts as the identity and the intensity epilogue
    // consumes the final matrix in-kernel
    if (!rays->p && !((flags & OLB_TF_POL_IDENTITY) && pol))
      return fail(OLB_ERR_INVALID_ARG, "OLB_TF_POLARIZED needs rays.p");
    if (rays->p && !aligned16(rays->p)) return fail(OLB_ERR_ALIGNMENT, "rays.p not 16-byte aligned");
    return launch_feat<T, 1>(a, features, stream);
  }
  const bool closed_form = (features & ~FEAT_ROT) == 0;
  // fp32: 4 rays/thread closed form, 2 with even/odd aspheres, 1 with the polynomial-family Newton surfaces
  // (2 rays/thread only adds register pressure to their long Newton loops)
  const bool poly_newton = (wh->hints & (int32_t)HINT_POLY_NEWTON) != 0;
  const int rpt = sizeof(T) == 4 ? (closed_form ? 4 : (poly_newton ? 1 : 2)) : (closed_form ? 2 : 1);
  if constexpr (sizeof(T) == 4) {
    if (rpt >= 4 && vec_ok) return launch_feat_cf<T, 4>(a, features, stream);
    if (rpt >= 2 && rec_stride_ok2) return launch_feat<T, 2>(a, features, stream);
  } else {
    if (rpt >= 2 && vec_ok) return launch_feat<T, 2>(a, features, stream);
  }
  return launch_feat<T, 1>(a, features, stream);
}

// ---- ray-aiming solve (OlbAimCall, olb_aim.cuh) ----------------------------------------------
struct AimArgs {
  const unsigned char* blob;
  int32_t blob_bytes;
  int32_t first, last;
  int32_t max_iter, infinite;
  int64_t n_rays;
  void* x; void* y; void* z; void* L; void* M; void* N; const void* w;
  const void* px; const void* py;
  double r_stop, J_factor, tol_sq;
  int32_t* status;
};

// One ray per thread, grid-stride; the table is staged in shared memory as in trace_kernel.  Writes only the two
// solved parameters of each ray and the status word.
template <typename T, uint32_t FEAT>
__global__ void __launch_bounds__(BLOCK) aim_kernel(const __grid_constant__ AimArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem);
  unsigned char* tab = smem + 16;
  stage_table(tab, a.blob, (uint32_t)a.blob_bytes, bar);
  const PrepHeader* H = reinterpret_cast<const PrepHeader*>(tab);
  const PrepSurface<T>* surf = reinterpret_cast<const PrepSurface<T>*>(tab + sizeof(PrepHeader));
  const T* pool = reinterpret_cast<const T*>(surf + H->n_surf);
  const T* wl = pool + H->pad[0];
  const T r_stop = (T)a.r_stop, Jf = (T)a.J_factor, tol_sq = (T)a.tol_sq;
  const bool inf = a.infinite != 0;
  int status = 0;
  for (int64_t k = (int64_t)blockIdx.x * BLOCK + threadIdx.x; k < a.n_rays; k += (int64_t)gridDim.x * BLOCK) {
    T x = ((const T*)a.x)[k], y = ((const T*)a.y)[k], z = ((const T*)a.z)[k];
    T L = ((const T*)a.L)[k], M = ((const T*)a.M)[k], N = ((const T*)a.N)[k];
    const int widx = H->n_wl > 1 ? aim_widx<T>(wl, H->n_wl, ((const T*)a.w)[k]) : 0;
    const T tx = o_mul_nc(((const T*)a.px)[k], r_stop), ty = o_mul_nc(((const T*)a.py)[k], r_stop);
    status |= aim_ray<T, FEAT>(surf, pool, a.first, a.last, x, y, z, L, M, N, widx, tx, ty, Jf, tol_sq, a.max_iter, inf);
    if (inf) { ((T*)a.x)[k] = x; ((T*)a.y)[k] = y; }
    else { ((T*)a.L)[k] = L; ((T*)a.M)[k] = M; }
  }
  if (status != 0) atomicOr(a.status, status);
}

template <typename T, uint32_t FEAT>
static int launch_aim(const AimArgs& a, cudaStream_t stream) {
  auto kern = aim_kernel<T, FEAT>;
  const size_t smem = 16 + (size_t)a.blob_bytes;
  static thread_local int cached_dev = -1;
  static thread_local int num_sms = 0;
  static thread_local int blocks_per_sm = 0;
  static thread_local size_t cached_smem = 0;
  int dev = 0;
  OLB_CUDA(cudaGetDevice(&dev));
  if (dev != cached_dev || smem != cached_smem) {
    if (smem > 48 * 1024) OLB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    OLB_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
    OLB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, kern, BLOCK, smem));
    if (blocks_per_sm < 1) return fail(OLB_ERR_CUDA, "aim kernel does not fit on an SM (table too large?)");
    cached_dev = dev;
    cached_smem = smem;
  }
  // one resident wave at most: each CTA stages the table once and then strides over the rays
  int64_t grid = (a.n_rays + BLOCK - 1) / BLOCK;
  const int64_t wave = (int64_t)num_sms * blocks_per_sm;
  if (grid > wave) grid = wave;
  kern<<<(unsigned)grid, BLOCK, smem, stream>>>(a);
  OLB_CUDA(cudaGetLastError());
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return OLB_OK;
}

template <typename T>
static int aim_impl(const OlbDeviceTable* wh, const OlbAimCall& c, cudaStream_t stream) {
  if (!wh || wh->magic != WS_MAGIC || !wh->workspace)
    return fail(OLB_ERR_INVALID_ARG, "table handle was not initialised by olb_table_upload");
  if (wh->n_systems > 1) return fail(OLB_ERR_UNSUPPORTED, "ray aiming on a batched table is not built");
  if (c.n_rays < 0) return fail(OLB_ERR_INVALID_ARG, "n_rays < 0");
  if (c.first < 0 || c.last > wh->n_surfaces || c.first >= c.last) return fail(OLB_ERR_INVALID_ARG, "bad surface range");
  if (c.max_iter < 0) return fail(OLB_ERR_INVALID_ARG, "max_iter < 0");
  if (!c.status) return fail(OLB_ERR_INVALID_ARG, "status is NULL");
  const int variant = aim_variant(wh->features);
  if (variant < 0) return fail(OLB_ERR_UNSUPPORTED, "ray aiming through a BSDF surface, a polarizing coating or a Forbes Q-2D surface is not built");
  if (c.n_rays == 0) return OLB_OK;
  if (!c.rays) return fail(OLB_ERR_INVALID_ARG, "rays is NULL");
  const OlbRays& r = *c.rays;
  const void* req[] = {r.x, r.y, r.z, r.L, r.M, r.N, c.Px, c.Py};
  for (const void* p : req) {
    if (!p) return fail(OLB_ERR_INVALID_ARG, "a guess or pupil array is NULL");
    if (!aligned16(p)) return fail(OLB_ERR_ALIGNMENT, "guess or pupil array not 16-byte aligned");
  }
  if (wh->n_wl > 1) {
    if (!r.w) return fail(OLB_ERR_INVALID_ARG, "rays.w is NULL but the table has several wavelengths");
    if (!aligned16(r.w)) return fail(OLB_ERR_ALIGNMENT, "rays.w not 16-byte aligned");
  }
  AimArgs a{};
  a.blob = (const unsigned char*)wh->workspace + (sizeof(T) == 8 ? wh->off_f64 : wh->off_f32);
  a.blob_bytes = sizeof(T) == 8 ? wh->bytes_f64 : wh->bytes_f32;
  a.first = c.first; a.last = c.last; a.max_iter = c.max_iter; a.infinite = c.infinite ? 1 : 0;
  a.n_rays = c.n_rays;
  a.x = r.x; a.y = r.y; a.z = r.z; a.L = r.L; a.M = r.M; a.N = r.N; a.w = r.w;
  a.px = c.Px; a.py = c.Py;
  a.r_stop = c.r_stop; a.J_factor = c.J_factor; a.tol_sq = c.tol * c.tol;
  a.status = c.status;
  if (variant == AIM_CLOSED_FORM) return launch_aim<T, FEAT_ROT>(a, stream);
  if (variant == AIM_GENERAL) return launch_aim<T, AIM_FEAT_GENERAL>(a, stream);
  return launch_aim<T, AIM_FEAT_SUPERSET>(a, stream);
}

}  // namespace olb

// =============================================================================================
// C ABI
// =============================================================================================
using namespace olb;

extern "C" {

int olb_version(void) { return OLB_VERSION_MAJOR * 1000 + OLB_VERSION_MINOR; }

int olb_last_error(char* buf, int buf_len) {
  if (!buf || buf_len <= 0) return OLB_ERR_INVALID_ARG;
  snprintf(buf, (size_t)buf_len, "%s", g_last_error.c_str());
  return OLB_OK;
}

int64_t olb_launch_count(void) { return g_launches.load(); }

int64_t olb_table_workspace_bytes(const OlbTable* table) {
  if (!table) return fail(OLB_ERR_INVALID_ARG, "table is NULL");
  PrepResult pr = prepare_table(*table);
  if (!pr.error.empty()) return fail(OLB_ERR_TABLE, pr.error);
  return (int64_t)(64 + pr.blob_f64.size() + pr.blob_f32.size());
}

int olb_table_upload(const OlbTable* table, void* workspace, int64_t workspace_bytes, void* stream,
                     OlbDeviceTable* out) {
  if (!table || !workspace || !out) return fail(OLB_ERR_INVALID_ARG, "table, workspace or out is NULL");
  if (!aligned16(workspace)) return fail(OLB_ERR_ALIGNMENT, "workspace not 16-byte aligned");
  PrepResult pr = prepare_table(*table);
  if (!pr.error.empty()) return fail(OLB_ERR_TABLE, pr.error);
  OlbDeviceTable h{};
  h.workspace = workspace;
  h.workspace_bytes = workspace_bytes;
  h.magic = WS_MAGIC;
  h.features = pr.features;
  h.n_surfaces = table->n_surfaces;
  h.n_wl = table->n_wl;
  h.off_f64 = 64;
  h.bytes_f64 = (int32_t)pr.blob_f64.size();
  h.off_f32 = 64 + h.bytes_f64;
  h.bytes_f32 = (int32_t)pr.blob_f32.size();
  h.bwd_supported = pr.bwd_supported ? (pr.bwd_tables ? 2 : 1) : 0;
  h.bwd_slots = pr.total_gslots;
  h.n_systems = 1;
  h.hints = (int32_t)pr.hints;
  h.stride_f64 = h.bytes_f64;
  h.stride_f32 = h.bytes_f32;
  const int64_t need = 64 + (int64_t)h.bytes_f64 + h.bytes_f32;
  if (workspace_bytes < need)
    return fail(OLB_ERR_INVALID_ARG, "workspace too small (need " + std::to_string(need) + " bytes)");
  std::vector<unsigned char> staging((size_t)need, 0);
  std::memcpy(staging.data() + h.off_f64, pr.blob_f64.data(), pr.blob_f64.size());
  std::memcpy(staging.data() + h.off_f32, pr.blob_f32.data(), pr.blob_f32.size());
  cudaStream_t st = (cudaStream_t)stream;
  // Pageable source: cudaMemcpyAsync returns once the bytes have been staged for DMA, so `staging` may be freed
  // right away and no stream synchronisation is needed -- the trace launched next on `stream` is ordered behind
  // the copy.  (The synchronise that used to sit here cost every parameter change of an optimisation loop a full
  // pipeline drain.)
  OLB_CUDA(cudaMemcpyAsync(workspace, staging.data(), (size_t)need, cudaMemcpyHostToDevice, st));
  *out = h;
  return OLB_OK;
}

// ---- batched systems: B perturbed copies of one template ------------------------------------------------
static int build_batch(const OlbTable* tmpl, const double* params, int32_t n_systems, std::vector<unsigned char>& all64,
                       std::vector<unsigned char>& all32, OlbDeviceTable& h) {
  if (!tmpl || !params) return fail(OLB_ERR_INVALID_ARG, "template table or params is NULL");
  if (n_systems < 1 || n_systems > 65535) return fail(OLB_ERR_INVALID_ARG, "n_systems must be in [1, 65535]");
  BatchPrep bp = prepare_batch(*tmpl, params, n_systems);     // olb_prep.h (host logic, also checked on the CPU)
  if (!bp.error.empty()) return fail(bp.unsupported ? OLB_ERR_UNSUPPORTED : OLB_ERR_TABLE, bp.error);
  all64.swap(bp.all64);
  all32.swap(bp.all32);
  h.bytes_f64 = bp.bytes_f64; h.bytes_f32 = bp.bytes_f32;
  h.bwd_supported = 0; h.bwd_slots = 0;
  h.hints = (int32_t)bp.hints;
  h.magic = WS_MAGIC; h.features = bp.features; h.n_surfaces = tmpl->n_surfaces; h.n_wl = 1; h.n_systems = n_systems;
  h.stride_f64 = h.bytes_f64; h.stride_f32 = h.bytes_f32;
  h.off_f64 = 64; h.off_f32 = 64 + (int32_t)all64.size();
  return OLB_OK;
}

int64_t olb_table_batch_workspace_bytes(const OlbTable* template_table, int32_t n_systems) {
  if (!template_table) return fail(OLB_ERR_INVALID_ARG, "table is NULL");
  PrepResult pr = prepare_table(*template_table);
  if (!pr.error.empty()) return fail(OLB_ERR_TABLE, pr.error);
  // rotations may switch PSF bits but never the blob size
  return 64 + (int64_t)n_systems * (int64_t)(pr.blob_f64.size() + pr.blob_f32.size());
}

int olb_table_upload_batch(const OlbTable* template_table, const double* params, int32_t n_systems, void* workspace,
                           int64_t workspace_bytes, void* stream, OlbDeviceTable* out) {
  if (!workspace || !out) return fail(OLB_ERR_INVALID_ARG, "workspace or out is NULL");
  if (!aligned16(workspace)) return fail(OLB_ERR_ALIGNMENT, "workspace not 16-byte aligned");
  std::vector<unsigned char> a64, a32;
  OlbDeviceTable h{};
  int rc = build_batch(template_table, params, n_systems, a64, a32, h);
  if (rc) return rc;
  const int64_t need = 64 + (int64_t)a64.size() + (int64_t)a32.size();
  if (workspace_bytes < need) return fail(OLB_ERR_INVALID_ARG, "workspace too small");
  if (need > INT32_MAX) return fail(OLB_ERR_INVALID_ARG, "batched table larger than 2 GiB");
  h.workspace = workspace; h.workspace_bytes = workspace_bytes;
  cudaStream_t st = (cudaStream_t)stream;
  OLB_CUDA(cudaMemcpyAsync((unsigned char*)workspace + h.off_f64, a64.data(), a64.size(), cudaMemcpyHostToDevice, st));
  OLB_CUDA(cudaMemcpyAsync((unsigned char*)workspace + h.off_f32, a32.data(), a32.size(), cudaMemcpyHostToDevice, st));
  // (pageable sources: both calls return after staging; see olb_table_upload)
  *out = h;
  return OLB_OK;
}

int olb_trace_call_f32(const OlbDeviceTable* table, const OlbTraceCall* call, void* stream) {
  if (!call) return fail(OLB_ERR_INVALID_ARG, "call is NULL");
  return trace_impl<float>(table, *call, (cudaStream_t)stream);
}
int olb_trace_call_f64(const OlbDeviceTable* table, const OlbTraceCall* call, void* stream) {
  if (!call) return fail(OLB_ERR_INVALID_ARG, "call is NULL");
  return trace_impl<double>(table, *call, (cudaStream_t)stream);
}

int olb_aim_f32(const OlbDeviceTable* table, const OlbAimCall* call, void* stream) {
  if (!call) return fail(OLB_ERR_INVALID_ARG, "call is NULL");
  return aim_impl<float>(table, *call, (cudaStream_t)stream);
}
int olb_aim_f64(const OlbDeviceTable* table, const OlbAimCall* call, void* stream) {
  if (!call) return fail(OLB_ERR_INVALID_ARG, "call is NULL");
  return aim_impl<double>(table, *call, (cudaStream_t)stream);
}

int olb_trace_bwd_f32(const OlbDeviceTable* table, int32_t first, int32_t last, const OlbRays* rays_in,
                      const OlbRecords* rec, const OlbRecords* grad_rec, const OlbRays* grad_rays_in,
                      double* grad_params, double* grad_tables, int64_t n_rays, uint64_t grad_row_mask, void* stream) {
  return trace_bwd_impl<float>(table, first, last, rays_in, rec, grad_rec, grad_rays_in, grad_params, grad_tables, n_rays,
                               grad_row_mask, (cudaStream_t)stream);
}
int olb_trace_bwd_f64(const OlbDeviceTable* table, int32_t first, int32_t last, const OlbRays* rays_in,
                      const OlbRecords* rec, const OlbRecords* grad_rec, const OlbRays* grad_rays_in,
                      double* grad_params, double* grad_tables, int64_t n_rays, uint64_t grad_row_mask, void* stream) {
  return trace_bwd_impl<double>(table, first, last, rays_in, rec, grad_rec, grad_rays_in, grad_params, grad_tables, n_rays,
                                grad_row_mask, (cudaStream_t)stream);
}

// ---- host-buffer end-to-end path ---------------------------------------------------------------
// scratch layout: HOST_SLOTS slots x 9 arrays (x,y,z,L,M,N,i,w,opd) x chunk elements
int64_t olb_host_scratch_bytes(int32_t elem_size, int64_t chunk_rays) {
  if ((elem_size != 4 && elem_size != 8) || chunk_rays < 1) return fail(OLB_ERR_INVALID_ARG, "bad scratch query");
  const int64_t chunk_al = (chunk_rays + 63) & ~int64_t(63);
  return (int64_t)HOST_SLOTS * 9 * chunk_al * elem_size;
}

}  // extern "C"

template <typename T>
static int trace_host_impl(const OlbDeviceTable* table, int32_t first, int32_t last, const OlbPupilLaunch* launch,
                           const OlbRays* h_in, const OlbRays* h_out, const OlbRecords* rec, int64_t n_rays,
                           int64_t chunk, void* scratch, int64_t scratch_bytes, uint32_t flags, int32_t* status) {
  if (!table || table->magic != WS_MAGIC) return fail(OLB_ERR_INVALID_ARG, "table handle was not initialised");
  const OlbDeviceTable& wh = *table;
  OlbRays pupil_in{};
  if (launch) {   // slots 0/1 carry Px/Py instead of x/y; the rest of the launch state is generated on the device
    if (!launch->Px || !launch->Py) return fail(OLB_ERR_INVALID_ARG, "launch.Px / launch.Py is NULL");
    if ((launch->Hx == nullptr) != (launch->Hy == nullptr)) return fail(OLB_ERR_INVALID_ARG, "launch.Hx and launch.Hy go together");
    // per-ray field points (trace_generic's call shape): two more host arrays ride in the z / L slots
    pupil_in.x = const_cast<void*>(launch->Px); pupil_in.y = const_cast<void*>(launch->Py);
    pupil_in.z = const_cast<void*>(launch->Hx); pupil_in.L = const_cast<void*>(launch->Hy);
    pupil_in.w = h_out ? h_out->w : nullptr;
    h_in = &pupil_in;
  }
  if (!h_in || !h_out || !scratch) return fail(OLB_ERR_INVALID_ARG, "NULL argument");
  if (chunk < 1) return fail(OLB_ERR_INVALID_ARG, "chunk_rays < 1");
  if (scratch_bytes < olb_host_scratch_bytes((int)sizeof(T), chunk)) return fail(OLB_ERR_INVALID_ARG, "scratch too small");
  if (!aligned16(scratch)) return fail(OLB_ERR_ALIGNMENT, "scratch not 16-byte aligned");
  const bool need_w = wh.n_wl > 1;
  const void* in[9] = {h_in->x, h_in->y, h_in->z, h_in->L, h_in->M, h_in->N, h_in->i, h_in->w, nullptr};
  void* out[9] = {h_out->x, h_out->y, h_out->z, h_out->L, h_out->M, h_out->N, h_out->i, nullptr, h_out->opd};
  for (int k = 0; k < 7; ++k)
    if ((!in[k] && !(launch && k >= 2)) || !out[k]) return fail(OLB_ERR_INVALID_ARG, "a required host ray array is NULL");
  if (!out[8]) return fail(OLB_ERR_INVALID_ARG, "h_out.opd is NULL");
  if (need_w && !in[7]) return fail(OLB_ERR_INVALID_ARG, "h_in.w is NULL but the table has several wavelengths");

  const int64_t chunk_al = (chunk + 63) & ~int64_t(63);
  constexpr int NS = HOST_SLOTS;
  T* slot[NS][9];
  for (int s = 0; s < NS; ++s)
    for (int k = 0; k < 9; ++k) slot[s][k] = (T*)scratch + ((int64_t)s * 9 + k) * chunk_al;

  // The NS copy / compute streams are created once per (host thread, device) and reused by every later call:
  // creating and destroying them per call cost ~60 us and a device-wide synchronisation point each time.
  static thread_local cudaStream_t tl_streams[16][NS];
  static thread_local bool tl_have[16] = {};
  int dev = 0;
  OLB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 16) return fail(OLB_ERR_INVALID_ARG, "device ordinal beyond 15");
  if (!tl_have[dev]) {
    for (int s = 0; s < NS; ++s) OLB_CUDA(cudaStreamCreateWithFlags(&tl_streams[dev][s], cudaStreamNonBlocking));
    tl_have[dev] = true;
  }
  cudaStream_t* st = tl_streams[dev];
  int result = OLB_OK;
  int64_t done = 0;
  int ci = 0;
  while (done < n_rays) {
    const int64_t m = (n_rays - done) < chunk ? (n_rays - done) : chunk;
    const int s = ci % NS;
    cudaStream_t q = st[s];
    // slot reuse is ordered by the stream itself (chunk ci and ci+2 share stream + slot)
    const bool per_ray_fields = launch && launch->Hx != nullptr;
    for (int k = 0; k < 8; ++k) {
      if (k == 7 && !need_w) continue;
      if (launch && k >= 2 && k != 7 && !(per_ray_fields && k <= 3)) continue;
      cudaError_t e = cudaMemcpyAsync(slot[s][k], (const T*)in[k] + done, (size_t)m * sizeof(T), cudaMemcpyHostToDevice, q);
      if (e != cudaSuccess) { result = fail(OLB_ERR_CUDA, cudaGetErrorString(e)); break; }
    }
    if (result) break;
    cudaError_t e = cudaSuccess;
    if (!launch) e = cudaMemsetAsync(slot[s][8], 0, (size_t)m * sizeof(T), q);   // (pupil launch: opd starts at 0 in-kernel)
    if (e != cudaSuccess) { result = fail(OLB_ERR_CUDA, cudaGetErrorString(e)); break; }
    OlbRays d{};
    d.x = slot[s][0]; d.y = slot[s][1]; d.z = slot[s][2]; d.L = slot[s][3]; d.M = slot[s][4]; d.N = slot[s][5];
    d.i = slot[s][6]; d.w = need_w ? slot[s][7] : nullptr; d.opd = slot[s][8];
    OlbRecords rr{};
    const OlbRecords* rp = nullptr;
    if (rec && rec->x) {
      rr = *rec;
      rr.x = (T*)rec->x + done; rr.y = (T*)rec->y + done; rr.z = (T*)rec->z + done;
      rr.L = (T*)rec->L + done; rr.M = (T*)rec->M + done; rr.N = (T*)rec->N + done;
      rr.intensity = (T*)rec->intensity + done; rr.opd = (T*)rec->opd + done;
      rp = &rr;
    }
    OlbPupilLaunch dl{};
    if (launch) {
      // the pupil slots double as the x / y outputs: read before written by the same thread
      dl = *launch;
      dl.Px = slot[s][0];
      dl.Py = slot[s][1];
      if (per_ray_fields) { dl.Hx = slot[s][2]; dl.Hy = slot[s][3]; }   // (read by each thread before it writes z / L)
    }
    OlbTraceCall call{};
    call.first = first; call.last = last; call.n_rays = m; call.flags = flags & ~uint32_t(OLB_TF_NO_FINAL);
    call.rays = &d; call.rec = rp; call.launch = launch ? &dl : nullptr; call.status = status;
    result = trace_impl<T>(&wh, call, q, done);   // BSDF draws: stream 0, ray indices of the whole host array
    if (result) break;
    for (int k = 0; k < 9; ++k) {
      if (k == 7) continue;
      e = cudaMemcpyAsync((T*)out[k] + done, slot[s][k], (size_t)m * sizeof(T), cudaMemcpyDeviceToHost, q);
      if (e != cudaSuccess) { result = fail(OLB_ERR_CUDA, cudaGetErrorString(e)); break; }
    }
    if (result) break;
    done += m;
    ++ci;
  }
  for (int s = 0; s < NS; ++s) {
    cudaError_t e = cudaStreamSynchronize(st[s]);
    if (e != cudaSuccess && !result) result = fail(OLB_ERR_CUDA, cudaGetErrorString(e));
  }
  return result;
}

extern "C" {

int olb_trace_host_f32(const OlbDeviceTable* table, int32_t first, int32_t last, const OlbPupilLaunch* launch,
                       const OlbRays* h_in, const OlbRays* h_out, const OlbRecords* rec, int64_t n_rays,
                       int64_t chunk_rays, void* dev_scratch, int64_t dev_scratch_bytes, uint32_t flags, int32_t* status) {
  return trace_host_impl<float>(table, first, last, launch, h_in, h_out, rec, n_rays, chunk_rays, dev_scratch,
                                dev_scratch_bytes, flags, status);
}
int olb_trace_host_f64(const OlbDeviceTable* table, int32_t first, int32_t last, const OlbPupilLaunch* launch,
                       const OlbRays* h_in, const OlbRays* h_out, const OlbRecords* rec, int64_t n_rays,
                       int64_t chunk_rays, void* dev_scratch, int64_t dev_scratch_bytes, uint32_t flags, int32_t* status) {
  return trace_host_impl<double>(table, first, last, launch, h_in, h_out, rec, n_rays, chunk_rays, dev_scratch,
                                 dev_scratch_bytes, flags, status);
}

}  // extern "C"
