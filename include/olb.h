/*
 * olb.h -- C ABI of libolb: the H100-native batched real-ray trace hot path.
 *
 * This is the drop-in boundary for ONE path of Optiland (reference under
 * Optiland v0.6.0): the per-surface loop
 *     SurfaceGroup.trace            optiland/surfaces/surface_group.py:245-257
 *       Surface.trace               optiland/surfaces/standard_surface.py:200-215
 *         Surface._trace_real       optiland/surfaces/standard_surface.py:232-248
 *         Surface._record_real      optiland/surfaces/standard_surface.py:260-274
 * The reference is pure Python and has no FFI below `optiland.backend`
 * (optiland/backend/__init__.py:100-190), so there is no existing C interface
 * to mirror; each entry point below names the reference function(s) whose work
 * it replaces.  The reference-side binding (ctypes) is shown in INTEGRATION.md.
 *
 * Rules of the ABI
 *   - plain pointers and sizes only; no torch / C++ types;
 *   - the CALLER owns every buffer (ray state, records, tables, workspace);
 *     the library allocates nothing that outlives a call;
 *   - every function returns OLB_OK (0) or a negative error code, and never
 *     throws; olb_last_error() returns a thread-local message;
 *   - numerical failure is IN-BAND, as in the reference: a missed surface or
 *     total internal reflection yields NaN coordinates that propagate
 *     (optiland/geometries/standard.py:132-135, optiland/rays/real_rays.py:179-180),
 *     vignetting sets intensity to 0 and the ray keeps propagating
 *     (optiland/rays/real_rays.py:154-161);
 *   - device pointers must be 16-byte aligned; `stream` is a cudaStream_t
 *     passed as void* (NULL = legacy default stream);
 *   - re-entrant per (stream, buffers); no global mutable state except the
 *     launch counter and the thread-local error string.
 */
#ifndef OLB_H_
#define OLB_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OLB_VERSION_MAJOR 0
#define OLB_VERSION_MINOR 3

/* ---- error codes ------------------------------------------------------- */
#define OLB_OK                 0
#define OLB_ERR_INVALID_ARG   -1   /* NULL pointer, bad range, bad enum        */
#define OLB_ERR_UNSUPPORTED   -2   /* surface kind / feature not built         */
#define OLB_ERR_CUDA          -3   /* a CUDA runtime call failed               */
#define OLB_ERR_ALIGNMENT     -4   /* device pointer not 16-byte aligned       */
#define OLB_ERR_TABLE         -5   /* malformed surface table / pool offsets   */

/* ---- surface geometry kinds (OlbSurface.kind) --------------------------- */
#define OLB_GEOM_NOOP          0   /* ObjectSurface: no physics, still records
                                      (optiland/surfaces/object_surface.py:56-93) */
#define OLB_GEOM_PLANE         1   /* optiland/geometries/plane.py:72-109        */
#define OLB_GEOM_STANDARD      2   /* sphere/conic closed form
                                      optiland/geometries/standard.py:97-175     */
#define OLB_GEOM_EVEN_ASPHERE  3   /* Newton iteration on conic + sum C_i r^(2i+2)
                                      optiland/geometries/newton_raphson.py:119-168,
                                      optiland/geometries/even_asphere.py:93-140 */
#define OLB_GEOM_ZERNIKE       4   /* Newton iteration on conic + Zernike sum
                                      optiland/geometries/zernike.py:153-252     */
#define OLB_GEOM_ODD_ASPHERE   5   /* conic + sum C_i r^(i+1)
                                      optiland/geometries/odd_asphere.py         */
#define OLB_GEOM_POLYNOMIAL    6   /* conic + sum C_ij x^i y^j
                                      optiland/geometries/polynomial.py:105-155  */
#define OLB_GEOM_CHEBYSHEV     7   /* conic + sum C_ij T_i(x/norm_x) T_j(y/norm_y)
                                      optiland/geometries/chebyshev.py:126-191   */
#define OLB_GEOM_BICONIC       8   /* zx(x; Rx, kx) + zy(y; Ry, ky)
                                      optiland/geometries/biconic.py:72-160      */
#define OLB_GEOM_TOROIDAL      9   /* Y-Z conic + even polynomial curve rotated about an
                                      axis at distance R_rot: optiland/geometries/toroidal.py:87-232 */
#define OLB_GEOM_FORBES_QBFS  10   /* conic + phi(r) u^2 (1 - u^2) sum a_m Q_m(u^2), u = r / norm_radius, Forbes'
                                      slope-orthogonal Q polynomials: optiland/geometries/forbes/geometry.py:187-366 */
#define OLB_GEOM_GRID_SAG     11   /* bilinear interpolation of a table of sag values
                                      optiland/geometries/grid_sag.py:60-140 (see "Grid sag" below) */
#define OLB_MAX_GRID_ELEMENTS 8192 /* per table: sum over grid surfaces of nx + ny + nx * ny (e.g. 89 x 89) */

/*
 * Grid sag (GridSagGeometry).  Pool block at coef_off: x[nx], y[ny], sag[ny][nx] (row j holds y_j: sag_grid[j, i]);
 * aux0 = nx, n_coef = ny, nx, ny >= 2, coordinates finite and strictly increasing, sag values finite.  radius is inf
 * and conic 0; tol and max_iter are the geometry's.  The grids of one table are staged in shared memory with the rest
 * of it, so their prepared elements (nx + ny + nx ny per surface) are capped at OLB_MAX_GRID_ELEMENTS per table.
 * The reference's semantics, reproduced exactly:
 *   cell      i = searchsorted(x, px, side="right") - 1 clamped to [0, nx - 2], j likewise: a point exactly on a node
 *             takes the cell to its upper right, and the upper edge px == x[nx-1] is inside, in the last cell (the
 *             on-axis chief ray of a grid with a node at 0 sits on that node, where the slope is discontinuous);
 *   value     bilinear, tx = (px - x_i) / (x_{i+1} - x_i), ty likewise; the SAG is NaN outside [x_0, x_{nx-1}] x
 *             [y_0, y_{ny-1}], the SLOPES are not: they are extrapolated from the clamped cell;
 *   distance  Newton from t = 0 at the incoming point (no base conic): t += -f / f', f = sag - z,
 *             f' = sx L + sy M - N (no guard on f' = 0).  An iterate that leaves the grid makes t NaN for good; a
 *             final out-of-grid test of the intercept also gives NaN;
 *   normal    (-sx, -sy, 1) / |.| -- the opposite sign to every other geometry's (fx, fy, -1).  Refraction and
 *             reflection align it with the ray and do not see the sign; a phase profile on a grid substrate does.
 * Convergence: the reference stops when the LARGEST |dt| over all rays is below tol (and, since max propagates NaN,
 * never while some ray is NaN).  The kernel iterates each ray until its own |dt| < tol (floored at the rounding noise of
 * t), applies that step, then takes one more (polishing) step, never more than max_iter steps in all.  Inside a cell
 * f is a quadratic in t, so Newton converges quadratically: once |dt| < tol the remaining error is O(tol^2), and the
 * extra steps the reference gives converged rays while others still move change t by that much at most.  A ray that
 * never converges runs max_iter steps in both.
 * The adjoint treats the grid values as constants: gradients flow through the pose, the indices and every other
 * surface, not to the sag table.
 */

/* ---- OlbSurface.flags --------------------------------------------------- */
#define OLB_SF_REFLECT     (1u << 0)  /* is_reflective: rays.reflect instead of refract
                                         optiland/interactions/refractive_reflective_model.py:45-50 */
#define OLB_SF_ROTATED     (1u << 1)  /* R != identity (cs has tilts or tilted parents)      */
#define OLB_SF_APERTURE    (1u << 2)  /* surface.aperture is set (aper_off/aper_len valid)   */
#define OLB_SF_ABSORBING   (1u << 3)  /* some k1(lambda) > 0: Beer-Lambert attenuation
                                         optiland/propagation/homogeneous.py:45-53            */
#define OLB_SF_NORECORD    (1u << 4)  /* do not write this surface's record row              */

/* ---- coatings (OlbSurface.coating) -------------------------------------- */
#define OLB_COAT_NONE      0   /* rays.update() : identity for RealRays, basis change
                                  for PolarizedRays (optiland/interactions/base.py:111-128) */
#define OLB_COAT_SIMPLE    1   /* SimpleCoating: i *= T or R (optiland/coatings.py:164-237) */
#define OLB_COAT_FRESNEL   2   /* FresnelCoating (optiland/coatings.py:362-386,
                                  optiland/jones.py:71-117); needs polarized rays       */
#define OLB_COAT_THIN_FILM 3   /* ThinFilmCoating (coatings.py:544, thin_film/core.py)   */
#define OLB_COAT_POLARIZER 4   /* PolarizerCoating (coatings.py:418, JonesLinearPolarizer) */
#define OLB_COAT_RETARDER  5   /* RetarderCoating (coatings.py:450, JonesLinearRetarder) */
#define OLB_MAX_FILM_LAYERS 32
/*
 * THIN_FILM, POLARIZER and RETARDER are BaseCoatingPolarized coatings (coatings.py:285-331): a Jones matrix J
 * per ray, then P := O_out J O_in P with the basis s, p0, p1 of PolarizedRays.get_local_basis, i.e.
 *     M[a][b] = s_a (J00 s_b + J01 p0_b) + p1_a (J10 s_b + J11 p0_b) + J22 k1_a k0_b.
 * Like FresnelCoating they need polarized rays; for RealRays the update is a no-op.  Their block sits right
 * after the surface's media block, at pool[media_off + 5 * n_wl]:
 *   THIN_FILM : {L, d_1 .. d_L, then per wavelength j: n0, k0, ns, ks, (n_l, k_l) x L}, 0 <= L <=
 *               OLB_MAX_FILM_LAYERS, thicknesses d_l in micrometres (finite, >= 0); n0 + i k0 and ns + i ks are the
 *               stack's incident and substrate materials (ThinFilmStack, which the surface keeps equal to its own
 *               materials).  Per ray and polarization, the transfer-matrix method of thin_film/core.py:_tmm_coh
 *               with theta0 = aoi = arccos(clip(|n . k0|)) (the geometry's unaligned normal, the direction before
 *               the interaction) and Y = 0.002654418729832701:
 *                   X = nr^2 - k^2 - (n0~ sin theta0)^2 - 2 i nr k   (principal sqrt; n~ cos = sqrt(X))
 *                   eta_s = Y sqrt(X),  eta_p = Y^2 conj(n~)^2 / eta_s,  delta_l = 2 pi d_l / lambda sqrt(X_l)
 *                   [A B; C D] = prod_l [[cos delta, i sin delta / eta], [i eta sin delta, cos delta]]  (incident first)
 *                   denom = eta0 (A + etas B) + C + etas D  (1e-30 when |denom| == 0)
 *                   r = (eta0 A + eta0 etas B - C - etas D) / denom,   t = conj(2 eta0 / denom)
 *               (the conjugate on t is the reference's); J = diag(r_s, -r_p, -1) on reflection and
 *               diag(t_s, t_p, 1) on transmission.  A stack of zero layers is the bare interface of these formulas.
 *   POLARIZER : {ax, ay, az}, the normalised axis (JonesLinearPolarizer.axis).  u_in = (a.s, a.p0), u_out =
 *               (a.s, a.p1), each normalised (norm 0 -> 1); J = u_out u_in^T, J22 = 1.
 *   RETARDER  : {d, ax, ay, az}: retardance and normalised fast axis (JonesLinearRetarder.retardance / .axis).
 *               (us, up) = u_in;  J00 = e^{-id/2} us^2 + e^{id/2} up^2,  J01 = J10 = -2i sin(d/2) us up,
 *               J11 = e^{id/2} us^2 + e^{-id/2} up^2,  J22 = 1.
 * One deliberate difference: each layer's characteristic matrix is carried scaled by e^{-|Im delta|} (r does not see
 * the scale; t is multiplied back by e^{-sum |Im delta|}).  Where the reference's cosh / sinh overflow -- a thick,
 * strongly absorbing layer, e.g. 20 um with n = 0.2, k = 5 -- it returns NaN for every ray; the kernel returns the finite
 * limit (r of the opaque stack, t -> 0).  Below that range both agree to rounding.
 * The axis is dotted with s, p0 and p1 in the SURFACE'S LOCAL frame, although the reference's docstrings say
 * "global coordinates" -- the reference's behaviour, reproduced.  Polarizer and retarder act the same on
 * reflection and transmission.  A table with one of these coatings has bwd_supported = 0 and
 * olb_table_upload_batch rejects it (OLB_ERR_UNSUPPORTED).
 */

/* ---- interaction models (OlbSurface.interaction) ------------------------
 * 0 is the refractive / reflective model (optiland/interactions/refractive_reflective_model.py).  The
 * others are PhaseInteractionModel (optiland/interactions/phase_interaction_model.py:45-132), the generalized
 * Snell's law of a phase profile phi(x, y) on the surface, in the local frame, with k0 = 2 pi / (lambda * 1e-3):
 *     k_par = n1 k0 d - (n1 k0 d . n) n + grad phi - (grad phi . n) n,   R^2 = (n2 k0)^2 - |k_par|^2
 *     R^2 < 0 -> i := 0 and R^2 := 0 (evanescent: no NaN);  d := normalise(k_par +- sqrt(R^2) n)
 *     (+ refraction, - reflection; n2 := n1 for a reflective surface);  opd += -phi / k0;  i *= efficiency
 * with the geometry's normal n AS IT RETURNS IT (no alignment with the ray: on a curved substrate, whose
 * normal points to -z, transmitted rays leave backwards -- the reference's behaviour, reproduced).  The
 * coating step (SimpleCoating / FresnelCoating / the polarization update) follows as for refraction.
 * Block at pool[phase_off]: {efficiency, n_terms, params[n_terms]} with
 *   CONSTANT : n_terms = 1, {phi}                                 (phase/constant.py)
 *   LINEAR   : n_terms = 2, {Kx, Ky}: phi = Kx x + Ky y           (phase/linear_grating.py, its _K_x / _K_y)
 *   RADIAL   : 1 <= n_terms <= OLB_MAX_PHASE_TERMS, {a_1 .. a_n}: phi = sum_p a_p r^(2p)  (phase/radial.py)
 * 1 / k0 per wavelength is derived at upload from the table's wavelength list.  A table with a phase surface
 * has bwd_supported = 0 and olb_table_upload_batch rejects it (OLB_ERR_UNSUPPORTED).
 *
 * GRATING is the ruled grating, DiffractiveInteractionModel (optiland/interactions/diffractive_model.py:28-61,
 * RealRays.gratingdiffract), on OLB_GEOM_PLANE (PlaneGrating) or OLB_GEOM_STANDARD with a finite radius
 * (StandardGratingGeometry); the geometry intersects and has its normal exactly as Plane / StandardGeometry.
 * Block at pool[phase_off]: {1.0, 3, m, d, alpha} (the phase block's framing: "efficiency" exactly 1, three
 * terms): order m, period d in micrometres (finite, non-zero, either sign), groove orientation alpha in radians.
 * In the local frame, with the geometry's normal n and lambda in micrometres:
 *     grating vector f = (-sin alpha, cos alpha, 0)                     on a plane
 *                    f = -normalise(n x t), t = (1, tan alpha, dz/dx along the groove)   on a conic
 *     n := sign(d0 . n) n   (aligned with the ray as refraction does; sign(0) = 0)
 *     a = n1 d0 + g f,  g = m lambda sqrt(fx^2 + fy^2) / d
 *     T = a |n|^2 - (a . n) n,   Q = n2^2 |n|^2 - |a x n|^2
 *     d := normalise(+-T + sign(d) sqrt(Q) n)    (+ transmission, - reflection; n2 is material_post's index,
 *                                                 for a mirror the medium before the surface)
 * then the coating step with the unaligned normal, as for refraction.  Four behaviours of the reference are
 * reproduced as they are:
 *   1. a reflective grating returns the NEGATIVE of the physical reflected direction (the next surface is
 *      reached with t < 0; the OPD stays positive through |t n|);
 *   2. an evanescent order (Q < 0) gives NaN direction cosines and leaves the intensity unchanged (the NaN then
 *      travels in band, as a missed surface does);
 *   3. the grating adds no OPD term;
 *   4. SimpleCoating scales i by R or T; FresnelCoating and polarized rays update P from d0 and the new d.
 * A grating table also has bwd_supported = 0 and olb_table_upload_batch rejects it.
 */
#define OLB_INTERACT_REFRACT        0
#define OLB_INTERACT_PHASE_CONSTANT 1
#define OLB_INTERACT_PHASE_LINEAR   2
#define OLB_INTERACT_PHASE_RADIAL   3
#define OLB_INTERACT_GRATING        4
#define OLB_MAX_PHASE_TERMS        16

/* ---- aperture programs --------------------------------------------------
 * surface.aperture (optiland/physical_apertures/*.py) is flattened by the host
 * into a postfix program over the pool: each instruction is one opcode double
 * followed by its operands.  The evaluator keeps a small boolean stack; the
 * final value is `inside`; rays with inside == false get i := 0
 * (optiland/physical_apertures/base.py:71-82).  NaN coordinates compare false,
 * so NaN rays are clipped, as in the reference.
 */
#define OLB_AP_RADIAL      1   /* r_max, r_min : r_min^2 <= x^2+y^2 <= r_max^2
                                  (radial.py:56-70)                                   */
#define OLB_AP_OFFSET_RADIAL 2 /* r_max, r_min, dx, dy   (offset_radial.py)           */
#define OLB_AP_RECT        3   /* x_min, x_max, y_min, y_max (rectangular.py)         */
#define OLB_AP_ELLIPSE     4   /* a, b, dx, dy           (elliptical.py)              */
#define OLB_AP_UNION       16  /* pops 2, pushes a | b   (base.py:259-340)            */
#define OLB_AP_INTERSECT   17  /* pops 2, pushes a & b                                */
#define OLB_AP_DIFFERENCE  18  /* pops 2, pushes a & ~b                               */

/* ---- trace flags (OlbTraceCall.flags, `flags` of olb_trace_host_*) -------- */
#define OLB_TF_POLARIZED   (1u << 0)  /* rays carry a 3x3 complex P matrix (OlbRays.p)  */
#define OLB_TF_POL_IDENTITY (1u << 2) /* with POLARIZED: P starts as identity, rays.p is output only */
#define OLB_TF_SHARED_INPUT (1u << 4) /* batched trace: every system traces the SAME rays_per_system launch rays */
#define OLB_TF_MOMENTS     (1u << 3)  /* accumulate OlbMoments over the traced batch (fused analysis
                                         epilogue, SURVEY.md 8f-2); see OlbTraceCall.moments         */
#define OLB_TF_MOMENTS_GLOBAL (1u << 5) /* moments of the GLOBAL (x, y) of the last traced surface instead of its local frame */
#define OLB_TF_MOMENTS_ALL (1u << 6)  /* moments over EVERY ray (no i > 0 / finite mask): a NaN ray makes the sums NaN, like
                                         be.mean over the record row in the rms_spot_size operand (operand/ray.py:337-341) */
#define OLB_TF_NO_FINAL    (1u << 1)  /* do not write the final state back into rays.x..opd:
                                         the caller takes it from the last record row (saves
                                         32-64 B/ray of HBM writes; needs rec)              */

#define OLB_MAX_SURFACES   64
#define OLB_MAX_WAVELENGTHS 16

/*
 * One optical surface, as the hot path sees it (data contract: SURVEY.md
 * Appendix B).  All real numbers are fp64 on the host side; the fp32 kernel
 * derives its own fp32 working copy on the device.  `pool` offsets are in
 * units of doubles into the table's pool array.
 *
 * Pose: (t, R) is the flattened effective transform of geometry.cs including
 * every parent reference_cs (optiland/coordinate_system.py:145-165):
 *     local  = R^T (global - t)      [CoordinateSystem.localize, :73-89]
 *     global = R local + t           [CoordinateSystem.globalize, :91-107]
 *
 * Media: for wavelength index j (0 <= j < n_wl of the table)
 *     pool[media_off + 0*n_wl + j] = n1  material_pre.n(lambda_j)
 *     pool[media_off + 1*n_wl + j] = n2  material_post.n(lambda_j)
 *     pool[media_off + 2*n_wl + j] = k1  material_pre.k(lambda_j)
 *     pool[media_off + 3*n_wl + j] = coating n1 (FresnelCoating.material_pre)
 *     pool[media_off + 4*n_wl + j] = coating n2 (FresnelCoating.material_post)
 * evaluated on the host by the reference's own material classes
 * (optiland/materials/base.py:98-149).  A thin-film, polarizer or retarder coating's block follows at
 * pool[media_off + 5*n_wl] (see OLB_COAT_THIN_FILM).
 */
typedef struct OlbSurface {
  int32_t kind;        /* OLB_GEOM_*                                          */
  uint32_t flags;      /* OLB_SF_*                                            */
  int32_t n_coef;      /* number of geometry coefficients / Zernike terms     */
  int32_t coef_off;    /* pool offset of the coefficient block (see below)    */
  int32_t aper_off;    /* pool offset of the aperture program                 */
  int32_t aper_len;    /* its length in doubles                               */
  int32_t max_iter;    /* Newton max_iter (newton_raphson.py:58-61)           */
  int32_t coating;     /* OLB_COAT_*                                          */
  int32_t media_off;   /* pool offset of the 5 x n_wl media block             */
  int32_t aux0;        /* polynomial: number of columns (y powers); grid: nx  */
  int32_t interaction; /* OLB_INTERACT_* (0: refractive / reflective)          */
  int32_t phase_off;   /* pool offset of the phase / grating block (see above) */
  double t[3];         /* effective translation                               */
  double R[9];         /* effective rotation, row-major                       */
  double radius;       /* geometry.radius (inf => plane branch of Standard)   */
  double conic;        /* geometry.k                                          */
  double tol;          /* Newton tol                                          */
  double coat_t;       /* SimpleCoating.transmittance                         */
  double coat_r;       /* SimpleCoating.reflectance                           */
  double norm_radius;  /* Zernike norm_radius / polynomial norm               */
} OlbSurface;          /* 192 bytes, multiple of 16                           */

/*
 * Coefficient blocks in the pool
 *   EVEN_ASPHERE : n_coef doubles C_0.. ; term i is C_i * r^(2(i+1))
 *   ODD_ASPHERE  : n_coef doubles C_0.. ; term i is C_i * r^(i+1)
 *   POLYNOMIAL   : n_coef = rows*cols doubles, C[i*cols+j] * x^i y^j
 *   CHEBYSHEV    : {norm_x, norm_y} then n_coef = rows*cols doubles C[i*cols+j] (aux0 = cols)
 *   BICONIC      : {radius_y, conic_y}; OlbSurface.radius / conic hold radius_x / conic_x
 *   TOROIDAL     : {radius_rot, conic_yz} then n_coef doubles alpha_i (term alpha_i y^(2(i+1)));
 *                  OlbSurface.radius holds the Y-Z base radius, OlbSurface.conic must be 0 (the
 *                  reference starts Newton from that SPHERE, toroidal.py:71-73)
 *   FORBES_QBFS  : n_coef doubles a_0 .. a_M (missing radial orders = 0); OlbSurface.norm_radius = rho_max.
 *                  The change of basis to the Clenshaw form (geometries/forbes/qpoly.py:56-115) happens in
 *                  olb_table_upload.
 *   ZERNIKE      : n_coef terms, each 4 doubles {n, m, c*N_nm (sag), c (derivative)}
 *                  -- the reference's derivative path omits the normalisation
 *                  constant N_nm (optiland/zernike/base.py:104-136 vs :42-68);
 *                  this quirk is reproduced, not fixed.
 */

/* The whole table: surfaces + pool + wavelength list. Host or device memory
 * (host for olb_table_upload: the library stages it; it is < 64 KiB). */
typedef struct OlbTable {
  const OlbSurface* surfaces;  /* n_surfaces entries                           */
  int32_t n_surfaces;
  int32_t n_wl;                /* number of distinct wavelengths, >= 1         */
  const double* wavelengths;   /* n_wl values (micrometres), exact ray.w values */
  const double* pool;          /* pool_len doubles                             */
  int32_t pool_len;
  int32_t reserved;
} OlbTable;

/*
 * Ray state, structure of arrays (RealRays: optiland/rays/real_rays.py:23-89).
 * All pointers are DEVICE pointers to n_rays elements of the kernel's element
 * type (float for *_f32, double for *_f64).  The trace updates x..opd in place
 * (the reference assigns new arrays to the same attributes).
 *   w       wavelength per ray; may be NULL when the table has n_wl == 1
 *   L0..N0  optional outputs: direction before the last interaction, in the
 *           last surface's local frame (real_rays.py:170-172); NULL to skip
 *   p       3x3 complex polarization matrix per ray (optiland/rays/polarized_rays.py:50);
 *           required with OLB_TF_POLARIZED.  Layout: a contiguous complex (N,3,3) array,
 *           i.e. [n_rays][3][3][2] elements with (Re, Im) interleaved -- exactly the memory
 *           of the reference's `rays.p` tensor (torch.view_as_real).  Updated in place; with
 *           OLB_TF_POL_IDENTITY the input is not read (P starts as the identity, as
 *           PolarizedRays.__init__ sets it).
 */
typedef struct OlbRays {
  void* x; void* y; void* z;
  void* L; void* M; void* N;
  void* i; void* w; void* opd;
  void* L0; void* M0; void* N0;
  void* p;
} OlbRays;

/*
 * Per-surface records (Surface._record_real, standard_surface.py:260-274; the
 * stacked views SurfaceGroup.x .. .intensity, surface_group.py:108-153).
 * Each pointer is a DEVICE pointer to a row-major (n_rows, row_stride) array;
 * row r receives the state after surface (first + r), in GLOBAL coordinates.
 * Any pointer may be NULL (that quantity is not recorded); rec itself may be
 * NULL (endpoint-only trace).
 */
typedef struct OlbRecords {
  void* x; void* y; void* z;
  void* L; void* M; void* N;
  void* intensity; void* opd;
  int64_t row_stride;   /* elements between consecutive rows (>= n_rays)      */
} OlbRecords;

/* Status word written by the kernels (device int32, caller-owned, optional). */
#define OLB_ST_CHEBYSHEV_RANGE (1 << 1) /* same for Chebyshev surfaces (chebyshev.py:230-244)            */
#define OLB_ST_ZERNIKE_RANGE (1 << 0)  /* some |x/norm_radius| or |y/norm_radius| > 1:
                                          the reference raises ValueError
                                          (optiland/geometries/zernike.py:254-266) */

#define OLB_ST_K_PARALLEL_X (1 << 2)    /* polarized intensity epilogue: a launch direction parallel to the x axis; the
                                          reference raises ValueError (optiland/rays/polarized_rays.py:216-218)     */

int olb_version(void);
/* Copies the calling thread's last error message into buf (NUL terminated). */
int olb_last_error(char* buf, int buf_len);

/*
 * Device-resident ("prepared") table handle.  Filled by olb_table_upload; a plain
 * caller-owned struct (the library keeps no registry): pass it to the trace entry points.
 * `workspace` is caller-allocated DEVICE memory of >= olb_table_workspace_bytes().
 */
typedef struct OlbDeviceTable {
  void* workspace;
  int64_t workspace_bytes;
  uint32_t magic;
  uint32_t features;       /* code paths the table needs (selects the kernel variant) */
  int32_t n_surfaces;
  int32_t n_wl;
  int32_t off_f64, bytes_f64;   /* fp64 blob inside workspace */
  int32_t off_f32, bytes_f32;   /* fp32 blob inside workspace */
  int32_t bwd_supported;        /* 1 if olb_trace_bwd_* covers every surface of the table; 2: covered, and the table has
                                   polynomial / Zernike / Chebyshev / Forbes surfaces, which need grad_tables */
  int32_t bwd_slots;            /* gradient accumulator slots per thread (backward kernel)   */
  int32_t n_systems;            /* 1, or the number of systems of a batched table            */
  int32_t stride_f64;           /* bytes between consecutive systems' fp64 / fp32 blobs      */
  int32_t stride_f32;
  int32_t hints;                /* launch-policy hints filled by the upload (never semantics) */
} OlbDeviceTable;

/* Bytes of device workspace needed for `table` (< 256 KiB). Negative = error code. */
int64_t olb_table_workspace_bytes(const OlbTable* table);

/*
 * Validate `table` (HOST memory), precompute everything that is uniform over rays
 * (flattened poses, surface-to-surface transforms, n1/n2 per wavelength, monomial form
 * of Zernike sums) and copy the result into `workspace` (DEVICE) on `stream`, asynchronously: work launched
 * on `stream` afterwards sees the table; other streams must be ordered behind it by the caller.  Replaces the
 * per-call Python walk over live surface objects; call again whenever a surface parameter changes.
 * A workspace that is too small is OLB_ERR_INVALID_ARG with the message "workspace too small (need N bytes)":
 * callers that skip olb_table_workspace_bytes (it prepares the table a second time) and pass a generous buffer
 * can retry on that.
 */
int olb_table_upload(const OlbTable* table, void* workspace, int64_t workspace_bytes,
                     void* stream, OlbDeviceTable* out);

/*
 * Launch state from pupil coordinates (the step immediately before the path, SURVEY.md 8f-1):
 * ParaxialRayAimer.aim_rays (optiland/rays/ray_aiming/paraxial.py:33-106) on top of
 * AngleField / ObjectHeight.get_ray_origins (optiland/fields/field_types/angle.py:17-58) makes every
 * launch ray of ONE field an affine function of its normalised pupil point (Px, Py):
 *     origin p0 = (origin0.x + origin_scale.x * Px, origin0.y + origin_scale.y * Py, origin0.z)
 *     target p1 = (target0.x + target_scale.x * Px, target0.y + target_scale.y * Py, target0.z)
 *     direction = (p1 - p0) / |p1 - p0|      ((0,0,1) when |p1 - p0| < 1e-9, paraxial.py:95-103)
 * with intensity `intensity` (no apodization: 1) and OPD 0.  The kernel evaluates this instead
 * of reading x,y,z,L,M,N,i,opd: 8 B/ray of input instead of 32 B/ray.
 */
typedef struct OlbPupilLaunch {
  const void* Px;            /* n_rays elements of the kernel's type (device; host for *_host_*) */
  const void* Py;
  double origin0[3];
  double origin_scale[2];
  double target0[3];
  double target_scale[2];
  double intensity;
  /* Per-ray FIELD coordinates (RealRayTracer.trace_generic, raytrace/real_ray_tracer.py:120-154: Hx, Hy, Px, Py
   * arrays).  With Hx / Hy non-NULL the origin and the target also move with the ray's field point:
   *     g(H) = tan(field_arg * H)  (field_mode 1: angle fields, field_arg = radians(max_field))
   *            H                   (field_mode 2: object-height fields)
   *     p0.x += origin_field[0] * g(Hx),  p0.y += origin_field[1] * g(Hy)
   *     p1.x += target_field[0] * g(Hx),  p1.y += target_field[1] * g(Hy)      (telecentric: target follows origin)
   * origin0 / target0 are then the H = 0 values.  NULL (field_mode 0): one field for all rays, as above. */
  const void* Hx;
  const void* Hy;
  int32_t field_mode;
  int32_t n_vig;             /* number of entries of `vig` (0: no vignetting factors), <= OLB_MAX_VIG_FIELDS              */
  double field_arg;
  double origin_field[2];
  double target_field[2];
  /* Vignetting factors per ray, looked up in-kernel (with Hx / Hy): FieldGroup.get_vig_factor
   * (optiland/fields/field_group.py:93-122) is a nearest-neighbour lookup over the DEFINED fields; vig[j] =
   * {Hx_j, Hy_j, vx_j, vy_j} (normalised field coordinates).  The ray's pupil point is scaled by (1 - vx, 1 - vy),
   * `vig_power` times in succession: RealRayTracer.trace_generic applies the factors once itself
   * (raytrace/real_ray_tracer.py:134-137) and the paraxial aimer once more (rays/ray_aiming/paraxial.py:72-96), so that
   * call shape passes 2.  Nearest = smallest squared distance in fp64, the first of equals (torch's cdist + argmin;
   * exact ties between two fields are resolved by rounding there and by a k-d tree in the NumPy backend). */
  int32_t vig_power;
  int32_t reserved;
  double vig[16][4];
} OlbPupilLaunch;
#define OLB_MAX_VIG_FIELDS 16

/*
 * Host-buffer end-to-end trace: HOST SoA in, HOST final ray state out, the
 * per-surface records stay on the device (rec, optional).  Rays are cut into
 * chunks; H2D copy, kernel and D2H copy of consecutive chunks overlap on three
 * streams.  `h_in` supplies x,y,z,L,M,N,i,w (opd ignored, starts at 0);
 * `h_out` receives x,y,z,L,M,N,i,opd.  Host buffers should be pinned.
 *   dev_scratch : device memory, >= olb_host_scratch_bytes(elem_size, chunk)
 * With `launch` (optional) the launch state is generated on the device from HOST pupil arrays instead
 * (launch->Px, launch->Py are host pointers; h_in may be NULL): 8 B/ray cross PCIe instead of 28-32 B/ray.
 * launch->Hx / Hy (host arrays, optional, together) give every ray its own field point --
 * RealRayTracer.trace_generic's call shape; for a table with several wavelengths the per-ray wavelengths are
 * then read from h_out->w (host).
 */
int64_t olb_host_scratch_bytes(int32_t elem_size, int64_t chunk_rays);
int olb_trace_host_f32(const OlbDeviceTable* table, int32_t first, int32_t last,
                       const OlbPupilLaunch* launch, const OlbRays* h_in, const OlbRays* h_out,
                       const OlbRecords* rec, int64_t n_rays, int64_t chunk_rays,
                       void* dev_scratch, int64_t dev_scratch_bytes, uint32_t flags,
                       int32_t* status);
int olb_trace_host_f64(const OlbDeviceTable* table, int32_t first, int32_t last,
                       const OlbPupilLaunch* launch, const OlbRays* h_in, const OlbRays* h_out,
                       const OlbRecords* rec, int64_t n_rays, int64_t chunk_rays,
                       void* dev_scratch, int64_t dev_scratch_bytes, uint32_t flags,
                       int32_t* status);

/*
 * Reverse mode (the backward pass of the autograd configuration; reference:
 * loss.backward() through the eager graph, optiland/optimization/optimizer/torch/base.py:96-156).
 * Given dLoss/d(record rows) it returns dLoss/d(launch state) and ACCUMULATES
 * dLoss/d(surface parameters) into grad_params: n_surfaces blocks of OLB_GP_COUNT doubles,
 *   [OLB_GP_TX..TZ] pose translation t, [OLB_GP_CURV] curvature 1/radius (d/dradius =
 *   -curv^2 * this), [OLB_GP_CONIC] k, [OLB_GP_N1] n1, [OLB_GP_N2] n2,
 *   [OLB_GP_COEF + j] even- / odd-asphere coefficient C_j (j < OLB_GP_MAX_COEF),
 *   [OLB_GP_R + 3 i + j] pose rotation matrix entry R_ij (tilted poses only; the caller chains it to the
 *   Euler angles, R = Rz Ry Rx, coordinate_system.py:121-143).
 * Everything is recomputed from the forward call's inputs and records (nothing else is
 * saved): `rays_in` is the launch state the forward call consumed (x,y,z,L,M,N,i), `rec` its
 * full records for the same [first, last).  grad_rec pointers may be NULL individually
 * (that quantity has zero gradient); grad_rays_in (x,y,z,L,M,N,i,opd) may be NULL.
 * Supported tables (OlbDeviceTable.bwd_supported): plane / standard / even- and odd-asphere geometry, any
 * pose (translation gradients, and for tilted poses dLoss/dR for the caller to chain to the tilt angles), any
 * aperture tree, no or simple coating, one wavelength per call (a batch that mixes wavelengths is split by the caller:
 * one table, one forward and one adjoint launch per wavelength, optiland_b200.plugin._trace_grad_per_wavelength);
 * otherwise OLB_ERR_UNSUPPORTED.  Rays that are NaN at a surface carry no gradient from that surface on: neither
 * through later rows nor through that surface's own row -- also when only part of the row is NaN, as for total
 * internal reflection (finite intercept, intensity and OPD, NaN direction); the rows in front of it still count.
 * grad_row_mask: bit r set = record row r of grad_rec may be non-zero (rows with a clear bit
 * are not read); pass ~0 when unknown.
 */
#define OLB_GP_TX 0
#define OLB_GP_TY 1
#define OLB_GP_TZ 2
#define OLB_GP_CURV 3
#define OLB_GP_CONIC 4
#define OLB_GP_N1 5
#define OLB_GP_N2 6
#define OLB_GP_COEF 7
#define OLB_GP_MAX_COEF 12
#define OLB_GP_R (OLB_GP_COEF + OLB_GP_MAX_COEF)   /* 9 entries, row-major: dLoss/dR of a tilted pose */
#define OLB_GP_COUNT (OLB_GP_R + 9)

/*
 * grad_tables: TABLE gradients for the polynomial families, required when OlbDeviceTable.bwd_supported == 2 (the
 * table holds OLB_GEOM_POLYNOMIAL / OLB_GEOM_ZERNIKE / OLB_GEOM_CHEBYSHEV surfaces of at most 12 x 12 monomials) and
 * ignored (may be NULL) when it is 1.  The adjoint goes through the
 * intersection by the implicit-function theorem with the TRUE gradient of the sag polynomial and through the normal with
 * the Hessian of the reference's slope polynomial (whose Zernike form omits the normalisation constants,
 * optiland/zernike/base.py:104-136).  grad_tables: n_surfaces blocks of OLB_GT_PER_SURFACE doubles, ACCUMULATED --
 *   [0 .. 143]   dLoss/dS_ij, S = the prepared sag table   (sag += sum_ij S_ij xn^i yn^j, entry i * 12 + j)
 *   [144 .. 287] dLoss/dD_ij, D = the prepared slope table
 * in which the user's coefficients are linear: polynomial C_ij = S_ij = D_ij; Zernike S = sum_k c_k N_k M_k,
 * D = sum_k c_k M_k with M_k the monomial expansion of the unit term (optiland_b200.table.zernike_monomials), so
 * dLoss/dc_k = N_k <M_k, dLoss/dS> + <M_k, dLoss/dD>  (Zernike variables: optiland/geometries/zernike.py:182-252);
 * Chebyshev: ONE table S = D = P with P_pq = sum_ij C_ij Tc[i][p] Tc[j][q] (Tc: monomial coefficients of T_n), its slope
 * entering the normal WITHOUT the factors 1 / norm_x, 1 / norm_y (the reference's form, chebyshev.py:171-181), so
 * dLoss/dC_ij = sum_pq Tc[i][p] (dLoss/dS + dLoss/dD)_pq Tc[j][q].
 * OLB_GEOM_FORBES_QBFS surfaces (at most 12 radial terms) also make bwd_supported 2 (they use none of the
 * table blocks): grad_params[OLB_GP_COEF + m] receives dLoss/db_m, b = the coefficients of the basis the Clenshaw
 * recurrence runs on (A b = a with the upper-banded f / g / h matrix of Forbes, Opt. Express 18, 19700 (2010),
 * eqs. A.14-A.16; optiland/geometries/forbes/qpoly.py:56-115), so dLoss/da = A^-T dLoss/db
 * (optiland_b200.autograd.forbes_basis_matrix).
 * OLB_GEOM_GRID_SAG surfaces make bwd_supported 2 as well (they use none of the table blocks): the adjoint goes through
 * the intersection with F = (sx, sy) at the hit point and through the normal with the Hessian of the bilinear cell,
 * sxx = syy = 0, sxy = ((z22 - z21) - (z12 - z11)) / (dx dy); the grid values are constants of the adjoint.
 */
#define OLB_GT_DIM 12
#define OLB_GT_PER_SURFACE (2 * OLB_GT_DIM * OLB_GT_DIM)
int olb_trace_bwd_f32(const OlbDeviceTable* table, int32_t first, int32_t last,
                      const OlbRays* rays_in, const OlbRecords* rec, const OlbRecords* grad_rec,
                      const OlbRays* grad_rays_in, double* grad_params, double* grad_tables, int64_t n_rays,
                      uint64_t grad_row_mask, void* stream);
int olb_trace_bwd_f64(const OlbDeviceTable* table, int32_t first, int32_t last,
                      const OlbRays* rays_in, const OlbRecords* rec, const OlbRecords* grad_rec,
                      const OlbRays* grad_rays_in, double* grad_params, double* grad_tables, int64_t n_rays,
                      uint64_t grad_row_mask, void* stream);

/*
 * Fused wavefront epilogue (SURVEY.md 8f-2, second half; OlbTraceCall.wavefront_ref / wavefront_out, optional,
 * together): instead of (or besides) records / the final state,
 * the trace writes per ray the OPD in waves against a spherical reference and the point where the ray meets
 * that sphere -- steps 4-5 of ChiefRayStrategy.compute_wavefront_data
 * (optiland/wavefront/strategy.py:179-190) on top of SphericalReference.path_length
 * (optiland/wavefront/reference_geometry.py:55-82):
 *   t = distance back along the ray from its image-surface intercept to the sphere (centre, radius);
 *   opd = ray.opd - n_image t + tilt . (Px, Py);  out.opd = (opd_ref - opd) / (wavelength_um * 1e-3);
 *   out.pupil_{x,y,z} = intercept - t (L, M, N);  out.intensity = ray intensity on the last surface.
 * `tilt` is the launch-plane term of _correct_tilt (strategy.py:93-139): (ux EPD/2, uy EPD/2) for an
 * infinite-object angle field, else 0 (it needs `launch`, the pupil samples).  The caller computes centre,
 * radius and opd_ref from the chief ray (one ordinary 1-ray trace).  Evaluated in fp64 for both element types.
 * `last` must be the image surface.  With OLB_TF_NO_FINAL and rec == NULL nothing else is written per ray.
 * Not built for batched systems.
 */
typedef struct {
  double center[3];
  double radius;
  double n_image;
  double tilt[2];
  double opd_ref;
  double wavelength_um;
} OlbWavefrontRef;
typedef struct {
  void* opd;        /* waves */
  void* pupil_x;
  void* pupil_y;
  void* pupil_z;
  void* intensity;
} OlbWavefrontOut;

/*
 * Polarized call shapes (config 5, OLB_TF_POLARIZED): PolarizedRays through the fused launch / the wavefront
 * epilogue, with the intensity epilogue of RealRayTracer.trace in-kernel (OlbTraceCall.pol).
 *
 * `pol` describes optic.polarization_state (optiland/rays/polarization_state.py:15-56) and asks for
 * PolarizedRays.update_intensity (optiland/rays/polarized_rays.py:122-133 with _get_3d_electric_field :204-233):
 *     p = (k x xhat) / |k x xhat|,  s = p x k          (k = the ray's LAUNCH direction)
 *     E0 = Ex e^{i phase_x} s + Ey e^{i phase_y} p ;  i = sum_states |P E0|^2 * i0 / n_states
 * (unpolarized light = the two orthogonal states (1, 0) and (0, 1), is_polarized == 0).  The updated intensity goes
 * to pol->intensity (device, n_rays) when given, otherwise into the final state's rays.i; the RECORD rows keep the
 * geometric intensity, as in the reference (only rays.i is updated, raytrace/real_ray_tracer.py:112-113).  The
 * wavefront epilogue's out.intensity receives the updated value.  A launch direction parallel to xhat sets
 * OLB_ST_K_PARALLEL_X (the reference raises).
 *
 * `pol` needs OLB_TF_POLARIZED in flags.  With `launch`, P starts as the identity (PolarizedRays.__init__, :50) and
 * rays.p is output only -- and may be NULL when pol is given (the P matrices are then not written at all: 72 / 144 B
 * per ray saved).  pol may be NULL (plain polarized trace: P matrices only).
 */
typedef struct OlbPolarization {
  int32_t is_polarized;     /* 0: unpolarized (mean of two orthogonal states); 1: (Ex, Ey, phase_x, phase_y) */
  int32_t reserved;
  double Ex, Ey;            /* normalised amplitudes (PolarizationState normalises them, :53-56)            */
  double phase_x, phase_y;  /* radians                                                                      */
  void* intensity;          /* optional device output, n_rays elements of the kernel's type                 */
} OlbPolarization;

/*
 * Batched many-systems tables (SURVEY.md 8f-4): B perturbed copies of one template system -- the shape of
 * tolerancing Monte-Carlo runs (optiland/tolerancing/monte_carlo.py) and of the BatchedRayEvaluator
 * (optiland/optimization/batched_evaluator.py:277-705), which the reference evaluates as B separate small
 * traces.  `params` (HOST): n_systems x n_surfaces blocks of OLB_BP_COUNT doubles with the ABSOLUTE values
 *   [OLB_BP_TX..TZ] pose translation and [OLB_BP_R .. +8] row-major rotation (the effective transform,
 *   coordinate_system.py:145-165, as in OlbSurface.t / .R), [OLB_BP_CURV] 1/radius, [OLB_BP_CONIC], [OLB_BP_N1], [OLB_BP_N2],
 *   [OLB_BP_COEF + j] even-asphere coefficients;
 * everything else (kinds, apertures, coatings, tolerances) comes from `template_table` (one wavelength).
 * Traced by olb_trace_call_* with OlbTraceCall.rays_per_system.
 */
#define OLB_BP_TX 0
#define OLB_BP_TY 1
#define OLB_BP_TZ 2
#define OLB_BP_R 3
#define OLB_BP_CURV 12
#define OLB_BP_CONIC 13
#define OLB_BP_N1 14
#define OLB_BP_N2 15
#define OLB_BP_COEF 16
#define OLB_BP_MAX_COEF 12
#define OLB_BP_COUNT (OLB_BP_COEF + OLB_BP_MAX_COEF)
int64_t olb_table_batch_workspace_bytes(const OlbTable* template_table, int32_t n_systems);
int olb_table_upload_batch(const OlbTable* template_table, const double* params, int32_t n_systems,
                           void* workspace, int64_t workspace_bytes, void* stream, OlbDeviceTable* out);

/*
 * Forward trace on device buffers: n_rays rays through surfaces [first, last) of the prepared table.
 * Replaces SurfaceGroup.trace(rays, skip=first) (surface_group.py:245-257) -- and, with last = first + 1, a single
 * Surface.trace as issued by the ray aimers (optiland/rays/ray_aiming/iterative.py:366).  Every optional stage
 * is switched on by its field of OlbTraceCall; every pointer may be NULL.  Asynchronous on `stream`.
 */
typedef struct OlbTraceCall {
  int32_t first, last;
  int64_t n_rays;
  uint32_t flags;             /* OLB_TF_*                                                                        */
  int32_t reserved;
  /* Device SoA (updated in place unless OLB_TF_NO_FINAL).  With `launch` it receives the final state
   * (x,y,z,L,M,N,i,opd; not needed with OLB_TF_NO_FINAL) and supplies `w` when the table has several wavelengths;
   * then, and whenever nothing would be read or written, it may be NULL. */
  const OlbRays* rays;
  const OlbRecords* rec;      /* optional record rows, row r <-> surface first + r                              */
  /* Launch state generated in-kernel from pupil coordinates (see OlbPupilLaunch) instead of read from rays.
   * Record row 0 of an object surface holds the generated launch state. */
  const OlbPupilLaunch* launch;
  /* Fused analysis epilogue (the step immediately after the path): moments of the ray intercepts on the
   * LAST traced surface, in that surface's local frame (what SpotDiagram transforms to,
   * optiland/analysis/spot_diagram/core.py:462-481), over rays with intensity > 0 and finite intercepts
   * (the mask of core.py:471-472), relative to `center`:
   *   m[0] = count, m[1] = sum (x - cx), m[2] = sum (y - cy), m[3] = sum ((x-cx)^2 + (y-cy)^2),
   *   m[4] = sum intensity, m[5] = sum opd, m[6] = sum opd^2,
   *   m[7] = number of rays with intensity > 0 whose intercept is NOT finite (the reference's mask keeps them, so its
   *          statistics are NaN whenever this is non-zero)
   * accumulated in fp64 INTO `moments` (device, 8 doubles; the caller zeroes it).  From these follow the
   * centroid, the RMS spot radius about the centroid or about `center` (rms_spot_radius, core.py:357-370)
   * and the OPD mean / variance without writing or re-reading any per-ray array: rec may be NULL and
   * with OLB_TF_NO_FINAL the trace writes nothing per ray.  moments != NULL implies OLB_TF_MOMENTS. */
  double center[2];
  double* moments;
  /* Batched table (olb_table_upload_batch; required, > 0, when the table holds several systems): system b
   * traces the ray segment [b * rays_per_system, (b+1) * rays_per_system), n_rays = n_systems * rays_per_system.
   * ONE launch, grid.y = system, each CTA stages its own system's table.  With OLB_TF_SHARED_INPUT (+ NO_FINAL)
   * all systems read the same rays_per_system launch rays.  rec rows have n_rays columns; `moments` receives
   * 8 doubles PER SYSTEM.  0: a single-system table. */
  int64_t rays_per_system;
  const OlbWavefrontRef* wavefront_ref;   /* wavefront epilogue (above), together with wavefront_out            */
  const OlbWavefrontOut* wavefront_out;
  const OlbPolarization* pol;             /* polarized intensity epilogue (above)                               */
  int32_t* status;            /* optional device int32, OR-ed with OLB_ST_* bits                                */
} OlbTraceCall;               /* 112 bytes                                                                      */
int olb_trace_call_f32(const OlbDeviceTable* table, const OlbTraceCall* call, void* stream);
int olb_trace_call_f64(const OlbDeviceTable* table, const OlbTraceCall* call, void* stream);

/*
 * Huygens-Fresnel PSF summation (SURVEY.md 8f-3; reference: NumbaSummation._huygens_fresnel_summation,
 * optiland/psf/huygens_fresnel_strategies.py:97-160, and TorchSummation.compute :183-273):
 *     field(P) = sum_Q amp_Q exp(-i k opd_Q) exp(i k R)/R * (1 + (P-Q).Q/(Rp R))/2,  psf = |field|^2
 * for n_image image points P and n_pupil pupil points Q (all DEVICE fp64 arrays, global coordinates, mm;
 * opd in mm; k = 2 pi / wavelength_mm).  pupil_amp_im may be NULL (real amplitudes); `field` (2*n_image
 * doubles, re/im interleaved) may be NULL; when given it also serves as scratch so that small images can
 * split the pupil sum over more CTAs.  Asynchronous on `stream`.
 */
int olb_huygens_psf_f64(const double* image_x, const double* image_y, const double* image_z, int64_t n_image,
                        const double* pupil_x, const double* pupil_y, const double* pupil_z,
                        const double* pupil_amp_re, const double* pupil_amp_im, const double* pupil_opd,
                        int32_t n_pupil, double wavelength_mm, double Rp, double* psf, double* field,
                        void* stream);

/*
 * FFT-PSF gridding (SURVEY.md 8f-3; reference: ScalarFFTPSF._generate_pupils, _pad_pupils, _compute_psf,
 * optiland/psf/fft.py:123-227) -- the element-wise passes on either side of the library FFT, one kernel each.
 *
 * olb_fft_pupil_*: the zero-PADDED complex pupil function of one wavelength, grid_size x grid_size (row-major, re/im
 * interleaved: torch.complex128 / complex64), written in one pass:
 *     P[pad + pr, pad + pc] = sqrt(intensity[k]) * exp(-i 2 pi opd_waves[k]),  k = cell_ray[pr * num_rays + pc] >= 0
 *     0 elsewhere;  pad = (grid_size - num_rays) / 2  (be.pad's pad_before, fft.py:216-225)
 * `cell_ray` (num_rays^2 DEVICE int32): index of the wavefront sample of each cell of the num_rays x num_rays pupil
 * grid, -1 outside the unit disk (the reference's masked assignment `P[R2 <= 1] = ...`, fft.py:141-157, in gather
 * form; the k-th in-disk cell in row-major order holds sample k).  opd_waves / intensity: n_samples DEVICE values
 * (WavefrontData.opd in waves, .intensity).  NaN / negative intensity propagate as in the reference.
 *
 * olb_fft_psf_accumulate_*: `amp` = fft2 of that array (the caller's library FFT); folds |amp|^2, the fftshift
 * (out[(i + n/2) % n] = in[i] on both axes) and the sum over wavelengths into one pass:
 *     psf[shift(r), shift(c)] = (first ? 0 : psf[...]) + |amp[r, c]|^2,  then  / div * mul  when `last`
 * (the reference's `sum(...) / norm_factor * 100`, fft.py:184-191).  psf: grid_size^2 DEVICE reals.
 * All asynchronous on `stream`; pupil / amp must be aligned to one complex element.
 */
int olb_fft_pupil_f64(const double* opd_waves, const double* intensity, int64_t n_samples, const int32_t* cell_ray,
                      int32_t num_rays, int32_t grid_size, double* pupil, void* stream);
int olb_fft_pupil_f32(const float* opd_waves, const float* intensity, int64_t n_samples, const int32_t* cell_ray,
                      int32_t num_rays, int32_t grid_size, float* pupil, void* stream);
int olb_fft_psf_accumulate_f64(const double* amp, int32_t grid_size, int32_t first, int32_t last, double div, double mul,
                               double* psf, void* stream);
int olb_fft_psf_accumulate_f32(const float* amp, int32_t grid_size, int32_t first, int32_t last, double div, double mul,
                               float* psf, void* stream);

/*
 * Incoherent irradiance binning (reference: IncoherentIrradiance._generate_field_data, non-differentiable branch,
 * optiland/analysis/irradiance.py:265-353): the weighted 2-D histogram of ray positions on a detector, in one pass.
 *
 *   local position  the ray point (x, y, z) in the detector surface's frame:
 *                     OLB_IRR_FRAME_TRANSLATE: x - t[0], y - t[1] subtracted in the RAY's precision, with t the values
 *                       the frame's x / y tensors hold (an unrotated frame without a parent: bit for bit what
 *                       CoordinateSystem.localize's translate gives);
 *                     OLB_IRR_FRAME_AFFINE: p_loc = R^T (p - t) in fp64, with (t, R) the frame's effective transform
 *                       (CoordinateSystem.get_effective_transform; R row-major); zero entries of R contribute nothing,
 *                       as a rotation by a zero angle is skipped.
 *   mask            a ray counts when i > 0 (NaN and negative power are dropped);
 *   bin             per axis searchsorted(edges, v, side="right") - 1 with v in its own precision compared against the
 *                   fp64 edges; v == the last edge goes into the last bin; v outside [edges[0], edges[n]], NaN and
 *                   +-inf are dropped (np.histogram2d);
 *   accumulate      hist[ix * ny + iy] += (double)i, in fp64 INTO `hist` (the caller zeroes it).
 *
 * x / y / z / i: n_rays DEVICE values of the entry point's precision.  x_edges (nx + 1) and y_edges (ny + 1) are HOST
 * fp64 arrays, finite and strictly increasing; the entry point copies them into the caller-owned DEVICE scratch
 * `edges` (nx + ny + 2 doubles) on `stream`.  Every argument is checked before any device call (NULL arrays, nx or
 * ny < 1, n_rays < 0, non-finite or non-increasing edges: OLB_ERR_INVALID_ARG).  Asynchronous on `stream`.
 */
#define OLB_IRR_FRAME_TRANSLATE 0
#define OLB_IRR_FRAME_AFFINE    1
/* Accumulation: AUTO picks from nx * ny and n_rays.  SHARED: per-CTA fp64 histograms in shared memory, flushed with one
 * atomic per non-zero bin (nx * ny <= 27648).  GLOBAL: fp64 atomics straight into `hist`.  Lanes of a warp that hit the
 * same bin are summed before their atomic on both paths. */
#define OLB_IRR_PATH_AUTO   0
#define OLB_IRR_PATH_SHARED 1
#define OLB_IRR_PATH_GLOBAL 2
typedef struct OlbIrradiance {
  const void* x;
  const void* y;
  const void* z;              /* read by OLB_IRR_FRAME_AFFINE only; may be NULL with OLB_IRR_FRAME_TRANSLATE        */
  const void* i;
  int64_t n_rays;
  int32_t frame;              /* OLB_IRR_FRAME_*                                                                   */
  int32_t nx, ny;
  int32_t path;               /* OLB_IRR_PATH_*: 0 lets the library choose (what callers want); the others force one
                                 accumulation path, to measure where the choice switches                           */
  double t[3];                /* frame origin                                                                      */
  double R[9];                /* OLB_IRR_FRAME_AFFINE: effective rotation, row-major                               */
  const double* x_edges;      /* HOST, nx + 1                                                                      */
  const double* y_edges;      /* HOST, ny + 1                                                                      */
  double* edges;              /* DEVICE scratch, nx + ny + 2                                                       */
  double* hist;               /* DEVICE, nx * ny, row ix = x bin                                                   */
} OlbIrradiance;              /* 184 bytes                                                                         */
int olb_irradiance_f32(const OlbIrradiance* call, void* stream);
int olb_irradiance_f64(const OlbIrradiance* call, void* stream);

/* Number of kernel launches issued by this process through the library
 * (for bench.py's gpu_launches claim). */
int64_t olb_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* OLB_H_ */
