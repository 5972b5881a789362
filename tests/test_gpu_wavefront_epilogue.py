"""The fused wavefront (OPD-map) epilogue (``OlbTraceCall.wavefront_*``, the ``wf_opd`` block at the end of
``trace_kernel``) on the GPU, in every kernel variant, both precisions and every call shape.

The epilogue's inputs are the final state the same kernel would store, so its reference is the SAME kernel: for every
case one launch writes the wavefront outputs and one launch of the same table, dtype, rays and kernel instance writes the
final state (``x .. N``, ``i``, ``opd``).  ``wavefront_point`` (csrc/olb_math.cuh) is then restated in ``np.longdouble``
on that final state (``_wavefront_ld``) and every output is held to a per-ray forward-error bound of the kernel's fp64
arithmetic (``_fp64_bound``).  In fp32 the bound adds what the epilogue may legitimately differ by: it reads the OPD as
``(double)hi + (double)lo`` while the stored record is ``fl32(hi + lo)``, and it rounds each output to fp32.  The
intensity must match bit for bit and NaN outputs must sit exactly where the reference has NaN.

Three reference spheres per fixture, from the fixture's fp64 records (``_spheres``): the chief-ray sphere (centred on the
image point of the central ray, through its intercept on the last surface before the image, as
``plugin.wavefront_chief_ray`` builds it), a sphere that about half the rays start inside (the ``t1 < 0 ? t2 : t1``
choice), and a laterally offset sphere that many rays miss (the ``d < 0 -> 0`` clamp).  Each branch is counted.

No tolerance here is picked: the fp64 bound comes from the operation count of ``wavefront_point``, the fp32-against-fp64
bound from the fixtures' achieved fp32 errors (``f32_achieved.json``, 3x), the moment sums from
``test_gpu_spot_moments``' summation bound.
"""
from __future__ import annotations

import ctypes as C
import json
import math
import os

import numpy as np
import pytest
import torch

from tests._util import GOLDEN
from tests.test_gpu_spot_moments import (BLOCK, MATRIX, _assert_sums, _case, _chain, _host_terms, _launch_scalars, _rays,
                                         _variant_rpt)

pytestmark = pytest.mark.gpu

U32, U64 = 2.0 ** -24, 2.0 ** -53
ULD = float(np.finfo(np.longdouble).eps) / 2      # the reference's own unit roundoff
UNIT = {torch.float32: U32, torch.float64: U64}
DTYPES = (torch.float32, torch.float64)
FIN = ("x", "y", "z", "L", "M", "N", "i", "opd")
WF = ("opd", "pupil_x", "pupil_y", "pupil_z", "intensity")
REC = ("x", "y", "z", "L", "M", "N", "intensity", "opd")

# fixture -> (RPT fp32, RPT fp64): the spot-moment matrix (every kernel variant that carries an epilogue; the epilogue
# needs the image surface, so only last = n_surfaces) plus the polarized variant, per-ray wavelengths, and simple coatings
# with non-radial apertures (a polynomial-family Newton table: one ray per thread)
EXTRA = {
    "cooke_polarized": (1, 1),
    "tilted_fold_polarized": (1, 1),
    "generic_polarized_c5": (1, 1),
    "dgauss_multiwl": (4, 2),
    "misc_apertures_coatings": (1, 1),
}
FIXTURES = {**{k: v[:2] for k, v in MATRIX.items()}, **EXTRA}
POLARIZED = {"cooke_polarized", "tilted_fold_polarized", "generic_polarized_c5"}


def _sizes(rpt):
    return sorted({1, 3, 5, 255, 257, BLOCK * rpt - 1, BLOCK * rpt + 1, 4099})


def _rpt(name, dtab, dtype):
    """RPT of the instance launched: polarized rays always run one ray per thread (launch_feat)."""
    return 1 if name in POLARIZED else _variant_rpt(dtab, dtype)


# ---- the reference: wavefront_point in long double, and its fp64 forward-error bound ---------------------------------

def _wavefront_ld(st, Px, Py, ref):
    """wavefront_point (olb_math.cuh) on the final state ``st`` (float64 arrays of the kernel's T values), evaluated in
    long double.  Returns the outputs, the intermediate magnitudes the error bound needs, and the branch masks."""
    L_ = np.longdouble
    with np.errstate(all="ignore"):
        x, y, z, L, M, N = (st[k].astype(L_) for k in ("x", "y", "z", "L", "M", "N"))
        c0, c1, c2 = (L_(v) for v in ref["center"])
        R, n = L_(ref["radius"]), L_(ref["n_image"])
        Lr, Mr, Nr = -L, -M, -N
        a = Lr * Lr + Mr * Mr + Nr * Nr
        b = 2 * (Lr * (x - c0) + Mr * (y - c1) + Nr * (z - c2))
        c = x * x + y * y + z * z - 2 * (x * c0 + y * c1 + z * c2) + c0 * c0 + c1 * c1 + c2 * c2 - R * R
        d = b * b - 4 * a * c
        miss = d < 0
        dc = np.where(miss, L_(0), d)
        sq = np.sqrt(dc)
        t1, t2 = (-b - sq) / (2 * a), (-b + sq) / (2 * a)
        inside = t1 < 0
        t = np.where(inside, t2, t1)
        tilt = (L_(ref["tilt"][0]) * Px.astype(L_) + L_(ref["tilt"][1]) * Py.astype(L_)) if Px is not None else L_(0) * x
        oimg = n * t
        o = st["opd"].astype(L_) - oimg + tilt
        inv_wl = L_(1.0 / (ref["wavelength_um"] * 1e-3))        # the launcher's double, exactly
        out = {"opd": (L_(ref["opd_ref"]) - o) * inv_wl, "pupil_x": x - t * L, "pupil_y": y - t * M,
               "pupil_z": z - t * N}
        f = lambda v: np.asarray(v, dtype=np.float64)  # noqa: E731
        mag = {"a": f(a), "b": f(b), "c": f(c), "d": f(dc), "t": f(t), "t1": f(t1), "t2": f(t2), "tilt": f(tilt),
               "oimg": f(oimg), "o": f(o), "B": f(2 * (abs(L * (x - c0)) + abs(M * (y - c1)) + abs(N * (z - c2)))),
               "C": f(x * x + y * y + z * z + 2 * (abs(x * c0) + abs(y * c1) + abs(z * c2)) + c0 * c0 + c1 * c1 + c2 * c2
                      + R * R),
               "T": f(abs(L_(ref["tilt"][0]) * Px.astype(L_)) + abs(L_(ref["tilt"][1]) * Py.astype(L_)))
               if Px is not None else np.zeros(x.shape)}
    hit = np.isfinite(mag["t"]) & ~f(miss).astype(bool)
    return out, mag, {"inside": hit & f(inside).astype(bool), "front": hit & ~f(inside).astype(bool),
                      "miss": f(miss).astype(bool), "start_inside": f(c < 0).astype(bool)}


def _fp64_bound(st, mag, ref, u, e_opd_in):
    """Per-ray forward-error bound of wavefront_point evaluated in arithmetic of unit roundoff u, as nvcc may contract
    it, on exact inputs except the OPD (off by e_opd_in).  Terms, from wavefront_point's operations:
      a = |D|^2: 3 roundings; b = 2 (D . (p - c)): the differences, the products and two sums, 5u of B = 2 sum|D_i (p-c)_i|;
      c: ten terms in one chain of at most ten roundings, 10u of C = sum of their magnitudes (the R^2 cancellation);
      d = b^2 - 4ac: the propagated e_b, e_a, e_c plus 3 roundings; the clamp d < 0 -> 0 is 1-Lipschitz;
      sqrt(d): |sqrt(d') - sqrt(d)| <= min(sqrt(e_d), e_d / sqrt(d)) (the first near d = 0), plus its rounding;
      t = (-b -+ sq) / 2a: the numerator's errors and rounding over 2a, and a's relative error; where |t1| is within its
      error of 0 the kernel may pick the other root: then |t2 - t1| more;
      opd_img = n t; o = opd - opd_img + tilt.P (2u of the tilt term); opd_wv = (opd_ref - o) inv_wl; tt = opd_img / n;
      p_out = p - tt D (2 roundings)."""
    A, B, C = mag["a"], mag["B"], mag["C"]
    b, c, d, t, t1, t2 = mag["b"], mag["c"], mag["d"], mag["t"], mag["t1"], mag["t2"]
    with np.errstate(all="ignore"):
        e_a = 3 * u * A
        e_b = 5 * u * B
        e_c = 10 * u * C
        e_d = 2 * np.abs(b) * e_b + e_b * e_b + 4 * (A * e_c + np.abs(c) * e_a + e_a * e_c) + 3 * u * (b * b + 4 * A * np.abs(c))
        e_sq = np.where(d > 0, np.minimum(np.sqrt(e_d), e_d / np.sqrt(d)), np.sqrt(e_d)) + u * np.sqrt(d)
        sq = np.sqrt(d)
        e_num = e_b + e_sq + u * (np.abs(b) + sq)
        e_t = e_num / (2 * (A - e_a)) + np.abs(t) * (e_a / (A - e_a) + u)
        e_t = np.where(np.abs(t1) <= e_t, e_t + np.abs(t2 - t1), e_t)
        n = float(ref["n_image"])
        e_oi = n * e_t + u * n * np.abs(t)
        e_T = 2 * u * mag["T"]
        e_o = e_opd_in + e_oi + e_T + 2 * u * (np.abs(st["opd"]) + np.abs(mag["oimg"]) + mag["T"])
        inv_wl = 1.0 / (ref["wavelength_um"] * 1e-3)
        wv = (float(ref["opd_ref"]) - mag["o"]) * inv_wl
        e = {"opd": (e_o + u * (abs(float(ref["opd_ref"])) + np.abs(mag["o"]))) * inv_wl + u * np.abs(wv)}
        e_tt = e_oi / n + u * np.abs(t)
        for k, p, D in (("pupil_x", "x", "L"), ("pupil_y", "y", "M"), ("pupil_z", "z", "N")):
            e[k] = np.abs(st[D]) * e_tt + 2 * u * (np.abs(st[p]) + np.abs(t * st[D]))
    return e


def _bound(st, mag, ref, dtype, Px):
    """The kernel's fp64 arithmetic (u64) + the reference's own (long double) + one rounding of each output to T; in
    fp32 the OPD the epilogue reads is hi + lo, within (u32 + u64) |opd_rec| of the stored record."""
    opd = np.abs(st["opd"])
    e_in = (U32 + U64) * (1 + U32) * opd if dtype == torch.float32 else 0.0 * opd
    e64 = _fp64_bound(st, mag, ref, U64, e_in)
    eld = _fp64_bound(st, mag, ref, ULD, 0.0 * opd)
    return {k: e64[k] + eld[k] for k in e64}


def _check(got, st, Px, Py, ref, dtype, ctx):
    """got (the epilogue's 5 outputs, host float64) against the long-double reference on the final state ``st``.
    Returns (branch masks, worst error / bound, the reference)."""
    want, mag, br = _wavefront_ld(st, Px, Py, ref)
    bnd = _bound(st, mag, ref, dtype, Px)
    worst = 0.0
    for k in WF[:4]:
        g = got[k]
        w = want[k]
        nan_w = np.isnan(np.asarray(w, dtype=np.float64))
        assert np.array_equal(np.isnan(g), nan_w), (ctx, k, int(np.isnan(g).sum()), int(nan_w.sum()))
        m = ~nan_w
        err = np.asarray(np.abs(g[m].astype(np.longdouble) - w[m]), dtype=np.float64)
        tol = bnd[k][m] + UNIT[dtype] * np.abs(g[m])
        bad = ~(err <= tol)
        assert not bad.any(), (ctx, k, int(bad.sum()), float(np.max(err[bad] / tol[bad])),
                               np.flatnonzero(m)[bad][:5].tolist())
        if m.any():
            worst = max(worst, float(np.max(err / np.where(tol > 0, tol, np.inf), initial=0.0)))
    assert np.array_equal(got["intensity"], st["i"], equal_nan=True), (ctx, "intensity")
    return br, worst, want, mag, bnd


# ---- launches through the C ABI (trace._trace) -----------------------------------------------------------------------

def _c_ref(ref):
    from optiland_b200 import _lib

    c = _lib.OlbWavefrontRef()
    c.center = (C.c_double * 3)(*[float(v) for v in ref["center"]])
    c.radius, c.n_image = float(ref["radius"]), float(ref["n_image"])
    c.tilt = (C.c_double * 2)(*[float(v) for v in ref["tilt"]])
    c.opd_ref, c.wavelength_um = float(ref["opd_ref"]), float(ref["wavelength_um"])
    return c


def _launch(dtab, dtype, n, src, wf=None, final=False, rec=False, mom=False, polarized=False, pol=False):
    """One olb_trace_call of ``n`` rays.  ``src`` = ("rays", {FIN + w: device tensors}) or ("pupil", (Px, Py, affine,
    w or None)).  Writes the wavefront outputs for sphere ``wf``, the final state (``final``), records (``rec``), moments
    (``mom``, masked local frame about (0, 0)); ``polarized``: PolarizedRays with P written; ``pol``: False (no
    intensity epilogue), None / "unpolarized" / (Ex, Ey, phase_x, phase_y), with pol.intensity written when there is no
    wavefront output.  Returns {"wf", "fin", "rec", "mom", "pol_i"} as device tensors."""
    from optiland_b200 import _lib
    from optiland_b200.trace import _c_launch, _c_polarization, _c_records, _out_buffer, _trace

    dev = dtab.device
    flags = 0 if final else _lib.TF_NO_FINAL
    c_rays = _lib.OlbRays()
    out = {}
    launch = None
    kind, data = src
    multi = dtab.table.n_wl > 1
    if kind == "rays":
        if final:                                   # the final state is written in place: give the launch a copy
            arr = {k: data[k].clone() for k in FIN}
            out["fin"] = arr
        else:
            arr = {k: data[k] for k in FIN}
        for k in FIN:
            setattr(c_rays, k, arr[k].data_ptr())
        if multi:
            c_rays.w = data["w"].data_ptr()
        if polarized:
            flags |= _lib.TF_POL_IDENTITY
    else:
        Px, Py, aff, w = data
        launch = _c_launch(aff, Px, Py)
        if multi:
            c_rays.w = w.data_ptr()
        if final:
            arr = {k: torch.empty(n, dtype=dtype, device=dev) for k in FIN}
            for k in FIN:
                setattr(c_rays, k, arr[k].data_ptr())
            out["fin"] = arr
    if polarized:
        flags |= _lib.TF_POLARIZED
        cd = torch.complex64 if dtype == torch.float32 else torch.complex128
        out["p"] = torch.empty((n, 3, 3), dtype=cd, device=dev)
        c_rays.p = torch.view_as_real(out["p"]).data_ptr()
    c_pol = None
    if pol is not False:
        if wf is None:
            out["pol_i"] = torch.empty(n, dtype=dtype, device=dev)
        c_pol = _c_polarization(pol, out.get("pol_i"))
    wavefront = None
    if wf is not None:
        buf = _out_buffer(5, 1, n, dtype, dev)[:, 0]
        wavefront = (_c_ref(wf), _lib.OlbWavefrontOut(*[buf[j].data_ptr() for j in range(5)]))
        out["wf"] = {k: buf[j, :n] for j, k in enumerate(WF)}
    c_rec = None
    last = dtab.table.num_surfaces
    if rec:
        rb = _out_buffer(8, last, n, dtype, dev)
        c_rec = _c_records(rb)
        out["rec"] = {k: rb[j, :, :n] for j, k in enumerate(REC)}
    moments = torch.zeros(8, dtype=torch.float64, device=dev) if mom else None
    _trace(dtab, dev, dtype, 0, last, n, flags, rays=c_rays, rec=c_rec, launch=launch, moments=moments,
           wavefront=wavefront, pol=c_pol)
    if mom:
        out["mom"] = moments
    return out


def _host(d):
    return {k: v.double().cpu().numpy() for k, v in d.items()}


# ---- fixtures: spheres, launch forms ---------------------------------------------------------------------------------

def _central_ray(c):
    """Index of the ray launched nearest the middle of the fixture's bundle (its chief ray, for one field)."""
    r = c.rays
    d = np.hypot(r["x"] - np.median(r["x"]), r["y"] - np.median(r["y"]))
    fin = np.isfinite(c.rec["x"][-1]) & np.isfinite(c.rec["x"][-2])
    return int(np.argmin(np.where(fin, d, np.inf)))


def _spheres(c):
    """Three reference spheres from the fixture's fp64 records (image row and the row before it)."""
    img = {k: c.rec[k][-1].astype(np.float64) for k in ("x", "y", "z", "L", "M", "N", "opd")}
    prev = np.stack([c.rec[k][-2] for k in ("x", "y", "z")])
    j = _central_ray(c)
    p = np.stack([img["x"], img["y"], img["z"]])
    D = np.stack([img["L"], img["M"], img["N"]])
    c1 = p[:, j]
    R1 = max(float(np.linalg.norm(c1 - prev[:, j])), 0.1 * c.scale)
    wl = float(np.median(c.rays["w"]))
    # opd_ref: the chief ray's own OPD to the sphere, so the map is the aberration (waves) on sphere 1
    chief_t = R1          # the chief ray starts at the centre: t = R / |D|
    opd_ref = float(img["opd"][j] - chief_t)
    fin = np.all(np.isfinite(p), axis=0) & np.all(np.isfinite(D), axis=0)
    s1 = {"center": c1, "radius": R1, "n_image": 1.0, "tilt": (0.0, 0.0), "opd_ref": opd_ref, "wavelength_um": wl}
    r2 = float(np.median(np.linalg.norm(p[:, fin] - c1[:, None], axis=0)))
    s2 = {"center": c1, "radius": max(r2, 1e-9 * c.scale), "n_image": 1.33, "tilt": (0.0, 0.0), "opd_ref": opd_ref,
          "wavelength_um": wl}
    q = p[:, fin] - R1 * D[:, fin]                  # where the rays are R1 back from the image
    qm = np.median(q, axis=1)
    s = float(np.median(np.linalg.norm(q - qm[:, None], axis=0)))
    s = max(s, 1e-6 * c.scale)
    s3 = {"center": qm + np.array([s, 0.0, 0.0]), "radius": s, "n_image": 1.0, "tilt": (0.0, 0.0), "opd_ref": opd_ref,
          "wavelength_um": wl}
    return [s1, s2, s3]


def _collimated(c):
    """A launch affine of a collimated beam along the fixture's mean direction that fills the disk the fixture's own
    rays fill on its launch plane."""
    r = c.rays
    cx, cy = 0.5 * (r["x"].max() + r["x"].min()), 0.5 * (r["y"].max() + r["y"].min())
    rad = 0.5 * max(np.ptp(r["x"]), np.ptp(r["y"]))
    d = np.array([r["L"].mean(), r["M"].mean(), r["N"].mean()])
    d /= np.linalg.norm(d)
    z0 = float(np.median(r["z"]))
    return {"origin0": (cx, cy, z0), "origin_scale": (rad, rad), "target0": (cx + d[0], cy + d[1], z0 + d[2]),
            "target_scale": (rad, rad), "intensity": 1.0}


def _affine(c):
    from optiland_b200.launch import pupil_affine

    sc = _launch_scalars(c)
    return pupil_affine(sc) if sc else _collimated(c)


def _pupil_samples(c, idx):
    """Pupil coordinates of the chosen rays: the fixture's own where it has them, otherwise a seeded disk sample."""
    if "x_Px" in c.z.files and _launch_scalars(c):
        return c.extra("Px")[idx].astype(np.float64), c.extra("Py")[idx].astype(np.float64)
    g = np.random.default_rng(idx.size)
    rr = np.sqrt(g.uniform(0, 1, idx.size))
    th = g.uniform(0, 2 * np.pi, idx.size)
    return rr * np.cos(th), rr * np.sin(th)


def _dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dtype)


def _ray_src(c, idx, dtype):
    rays = _rays(c, idx, dtype)
    d = {k: getattr(rays, k) for k in ("x", "y", "z", "L", "M", "N", "i", "opd")}
    d["w"] = rays.w
    return ("rays", d)


CASE_NAMES = list(FIXTURES)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("name", CASE_NAMES)
def test_wavefront_epilogue_equals_long_double_on_the_final_state(name, dtype):
    """Every size around the tile boundaries x call shape (ray arrays; pupil launch without and with a tilt; the same
    pupil rays permuted) x sphere: the epilogue == wavefront_point in long double on the same kernel's final state, to
    the derived bound.  In fp32, the OPD recovered from the outputs shows that the epilogue read the low half."""
    c, dtab = _case(name)
    rpt = _rpt(name, dtab, dtype)
    assert rpt == FIXTURES[name][0 if dtype == torch.float32 else 1], "the fixture no longer reaches its kernel variant"
    polarized = name in POLARIZED
    spheres = _spheres(c)
    aff = _affine(c)
    counts = np.zeros((3, 4), np.int64)      # sphere x (t1 < 0 -> t2, t1 >= 0, d < 0 clamped, ray starts inside)
    worst = 0.0
    low_seen = low_total = 0
    for n in _sizes(rpt):
        idx = np.random.default_rng(n).integers(0, c.n, size=n)
        Px, Py = _pupil_samples(c, idx)
        w = _dev(c.rays["w"][idx], dtype)
        perm = np.random.default_rng(n + 1).permutation(n)
        tilt = (0.05 * c.scale, -0.03 * c.scale)
        forms = [("rays", _ray_src(c, idx, dtype), None, None, (0.0, 0.0)),
                 ("pupil", ("pupil", (_dev(Px, dtype), _dev(Py, dtype), aff, w)), Px, Py, (0.0, 0.0)),
                 ("pupil_tilt", ("pupil", (_dev(Px, dtype), _dev(Py, dtype), aff, w)), Px, Py, tilt),
                 ("pupil_tilt_perm", ("pupil", (_dev(Px[perm], dtype), _dev(Py[perm], dtype), aff, w[perm].contiguous())),
                  Px[perm], Py[perm], tilt)]
        outs = {}
        for form, src, px, py, tl in forms:
            st = _host(_launch(dtab, dtype, n, src, final=True, polarized=polarized)["fin"])
            # the launch's own Px, Py as the kernel reads them (rounded to T)
            pxT = _dev(px, dtype).double().cpu().numpy() if px is not None else None
            pyT = _dev(py, dtype).double().cpu().numpy() if py is not None else None
            for si, sph in enumerate(spheres):
                ref = dict(sph, tilt=tl)
                got = _host(_launch(dtab, dtype, n, src, wf=ref, polarized=polarized)["wf"])
                ctx = (name, str(dtype), n, form, si)
                br, wr, want, mag, bnd = _check(got, st, pxT, pyT, ref, dtype, ctx)
                worst = max(worst, wr)
                counts[si] += [int(br[k].sum()) for k in ("inside", "front", "miss", "start_inside")]
                outs[(form, si)] = (got, bnd)
                if dtype == torch.float32 and si == 0:
                    s, t = _low_half(got, st, mag, ref, pxT, pyT, ctx)
                    low_seen += s
                    low_total += t
        # the permuted launch returns the same rays' outputs, permuted
        for si in range(3):
            g0, b0 = outs[("pupil_tilt", si)]
            g1, b1 = outs[("pupil_tilt_perm", si)]
            for k in WF[:4]:
                a, b = g0[k][perm], g1[k]
                assert np.array_equal(np.isnan(a), np.isnan(b)), (name, n, si, k)
                m = ~np.isnan(a)
                tol = b0[k][perm][m] + b1[k][m] + UNIT[dtype] * (np.abs(a[m]) + np.abs(b[m]))
                assert np.all(np.abs(a[m] - b[m]) <= tol), (name, n, si, k)
    total = counts[0, :3].sum()
    assert counts[0, 0] > 0, ("chief sphere: t1 < 0 selects t2", counts)
    assert 0 < counts[1, 3] < total and counts[1, 0] > 0, ("sphere 2: some rays start inside, t1 < 0", counts)
    assert counts[2, 2] > 0 and counts[2, 1] > 0, ("sphere 3: misses (d < 0) and hits", counts)
    msg = f"{name} {dtype}: worst error / bound {worst:.3e}; branches (t1<0, t1>=0, d<0, inside) {counts.tolist()}"
    if dtype == torch.float32:
        assert low_total > 0
        frac = low_seen / low_total
        msg += f"; fp32 low half observed on {frac:.3f} of {low_total} rays"
        assert frac > 0.5, msg
    print(msg)


def _low_half(got, st, mag, ref, Px, Py, ctx):
    """fp32: the OPD the epilogue used, recovered from its outputs, opd_ref - opd_wv / inv_wl + n t - tilt.P (t in long
    double from the same inputs), lies within (u32 + u64) |opd_rec| of the fp32 record plus the recovery noise -- the fp32
    rounding of the stored opd_wv in mm and the fp64 error of the epilogue itself -- and on most rays it differs from the
    record by more than that noise: the low half of the two-float OPD reached the epilogue.  Returns (rays where the
    difference was observed, rays checked)."""
    L_ = np.longdouble
    inv_wl = 1.0 / (ref["wavelength_um"] * 1e-3)
    wv = got["opd"]
    m = np.isfinite(wv) & np.isfinite(st["opd"]) & np.isfinite(mag["t"])
    tilt = mag["tilt"]
    rec_opd = (L_(ref["opd_ref"]) - wv.astype(L_) / L_(inv_wl) + L_(ref["n_image"]) * mag["t"].astype(L_)
               - tilt.astype(L_))
    diff = np.asarray(np.abs(rec_opd - st["opd"].astype(L_)), dtype=np.float64)
    e = _fp64_bound(st, mag, ref, U64, 0.0 * st["opd"])["opd"] + _fp64_bound(st, mag, ref, ULD, 0.0 * st["opd"])["opd"]
    noise = U32 * np.abs(wv) / inv_wl + e / inv_wl + float(ref["n_image"]) * 4 * ULD * np.abs(mag["t"])
    allowed = (U32 + U64) * (1 + U32) * np.abs(st["opd"]) + noise
    assert np.all(diff[m] <= allowed[m]), (ctx, "recovered OPD", float(np.max(diff[m] / allowed[m])))
    return int(np.count_nonzero(diff[m] > noise[m])), int(np.count_nonzero(m))


# ---- every output in one launch ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("name", CASE_NAMES)
def test_outputs_written_in_one_launch(name, dtype):
    """Records + final state + wavefront (+ moments) in one launch: the wavefront outputs bit-identical to the
    wavefront-only launch, records and final state bit-identical to the launch without the epilogue, moment counts equal
    to the moments-only launch and sums within test_gpu_spot_moments' summation bound of the records."""
    c, dtab = _case(name)
    rpt = _rpt(name, dtab, dtype)
    polarized = name in POLARIZED
    sph = _spheres(c)[0]
    last = c.table.num_surfaces
    for n in _sizes(rpt):
        idx = np.random.default_rng(n).integers(0, c.n, size=n)
        src = _ray_src(c, idx, dtype)
        wf = _launch(dtab, dtype, n, src, wf=sph, polarized=polarized)["wf"]
        plain = _launch(dtab, dtype, n, src, final=True, rec=True, polarized=polarized)
        both = _launch(dtab, dtype, n, src, wf=sph, final=True, rec=True, polarized=polarized)
        for k in WF:
            assert torch.equal(both["wf"][k].nan_to_num(7.0), wf[k].nan_to_num(7.0)), (name, n, k)
        for k in FIN:
            assert torch.equal(both["fin"][k].nan_to_num(7.0), plain["fin"][k].nan_to_num(7.0)), (name, n, k)
        for k in REC:
            assert torch.equal(both["rec"][k].nan_to_num(7.0), plain["rec"][k].nan_to_num(7.0)), (name, n, k)
        if polarized:
            continue            # the moments epilogue is not part of the polarized call shapes
        mom = _launch(dtab, dtype, n, src, mom=True)["mom"]
        full = _launch(dtab, dtype, n, src, wf=sph, final=True, rec=True, mom=True)
        for k in WF:
            assert torch.equal(full["wf"][k].nan_to_num(7.0), wf[k].nan_to_num(7.0)), (name, n, k)
        want = _host_terms(c, plain["rec"], last, (0.0, 0.0), False, False, dtype)
        k_chain = _chain(n, rpt)
        for m in (mom, full["mom"]):
            _assert_sums(m, want, k_chain, (name, n))
        assert float(full["mom"][0]) == float(mom[0]) and float(full["mom"][7]) == float(mom[7])


# ---- polarized rays: the intensity the epilogue writes ------------------------------------------------------------------

@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("name", sorted(POLARIZED))
def test_polarized_intensity_reaches_the_wavefront_outputs(name, dtype):
    """pol = NULL: out.intensity == the geometric final intensity, bit for bit.  pol unpolarized and one polarized
    state: out.intensity == pol.intensity of a launch without the epilogue, bit for bit (and differs from the
    geometric intensity on some rays, so the two cannot be confused); the other outputs still match the reference."""
    c, dtab = _case(name)
    sph = _spheres(c)[0]
    state = tuple(float(v) for v in c.extra("state")) if "x_state" in c.z.files else (1.0, 0.5, 0.0, 0.3)
    aff = _affine(c)
    for n in (257, 4099):
        idx = np.random.default_rng(n).integers(0, c.n, size=n)
        Px, Py = _pupil_samples(c, idx)
        w = _dev(c.rays["w"][idx], dtype)
        for src in (_ray_src(c, idx, dtype), ("pupil", (_dev(Px, dtype), _dev(Py, dtype), aff, w))):
            geo = _launch(dtab, dtype, n, src, final=True, polarized=True)["fin"]["i"]
            got = _launch(dtab, dtype, n, src, wf=sph, polarized=True)["wf"]["intensity"]
            assert torch.equal(got.nan_to_num(7.0), geo.nan_to_num(7.0)), (name, n, src[0], "pol NULL")
            for pol in ("unpolarized", state):
                ref_launch = _launch(dtab, dtype, n, src, final=True, polarized=True, pol=pol)
                pol_i = ref_launch["pol_i"]
                out = _host(_launch(dtab, dtype, n, src, wf=sph, polarized=True, pol=pol)["wf"])
                assert np.array_equal(out["intensity"], pol_i.double().cpu().numpy(), equal_nan=True), (name, n, pol)
                assert not torch.equal(pol_i, geo), (name, n, pol, "the intensity epilogue changed nothing")
                st = _host(ref_launch["fin"])
                assert np.array_equal(st["i"], out["intensity"], equal_nan=True)
                px = _dev(Px, dtype).double().cpu().numpy() if src[0] == "pupil" else None
                py = _dev(Py, dtype).double().cpu().numpy() if src[0] == "pupil" else None
                _check(out, st, px, py, sph, dtype, (name, n, pol))


# ---- fp32 against fp64: the "3x achieved" rule ------------------------------------------------------------------------

def _achieved(name):
    base = name.partition(":")[0]
    sub, case = os.path.split(base)
    path = os.path.join(GOLDEN, sub, "f32_achieved.json")
    if not os.path.exists(path):
        return None
    with open(path) as f:
        return json.load(f)["cases"].get(case)


F32_CASES = [n for n in CASE_NAMES if ":" not in n and _achieved(n) is not None]


def _partials(st, ref):
    """|d out / d in| of wavefront_point at the fp64 state, per input group (position, direction, OPD), for a ray
    that meets the sphere transversally: t solves |p - t D - c|^2 = R^2, so with q = p - t D, g = D.(q - c):
    dt/dp = (q - c) / g, dt/dD = -t (q - c) / g; opd_wv = (opd_ref - opd + n t) inv_wl; p_out = q."""
    x = np.stack([st["x"], st["y"], st["z"]])
    D = np.stack([st["L"], st["M"], st["N"]])
    c = np.asarray(ref["center"], dtype=np.float64)[:, None]
    want, mag, _ = _wavefront_ld(st, None, None, ref)
    t = mag["t"]
    q = x - t * D
    g = np.sum(D * (q - c), axis=0)
    dtdp = (q - c) / g
    dtdD = -t * (q - c) / g
    n, inv_wl = float(ref["n_image"]), 1.0 / (ref["wavelength_um"] * 1e-3)
    out = {"opd": (n * inv_wl * np.sum(np.abs(dtdp), axis=0), n * inv_wl * np.sum(np.abs(dtdD), axis=0),
                   inv_wl * np.ones_like(t))}
    for j, k in enumerate(("pupil_x", "pupil_y", "pupil_z")):
        # dq_j/dp_i = delta_ij - D_j dt/dp_i; dq_j/dD_i = -t delta_ij - D_j dt/dD_i
        delta = (np.arange(3)[:, None] == j).astype(np.float64)
        dp = np.sum(np.abs(delta - D[j] * dtdp), axis=0)
        dD = np.sum(np.abs(-t * delta - D[j] * dtdD), axis=0)
        out[k] = (dp, dD, np.zeros_like(t))
    return want, out


@pytest.mark.parametrize("name", F32_CASES)
def test_f32_epilogue_against_the_fp64_reference(name):
    """The fp32 epilogue on the fixture's rays against wavefront_point in long double on the fp64 oracle's final state
    (the reference's own records), chief-ray sphere: per ray within 3 sum_j |d out / d in_j| e_j, e_j the fixture's
    achieved fp32 position / direction / OPD errors, plus the fp32 rounding of the output; the intensity within 3x its
    achieved error.  Rays whose finite / NaN or i > 0 status flips between precisions: <= 2 %."""
    c, dtab = _case(name)
    e = _achieved(name)
    sph = _spheres(c)[0]
    st64 = {k: c.rec[r][-1].astype(np.float64) for k, r in zip(FIN, REC)}
    n = c.n
    idx = np.arange(n)
    got = _host(_launch(dtab, torch.float32, n, _ray_src(c, idx, torch.float32), wf=sph,
                        polarized=name in POLARIZED)["wf"])
    want, part = _partials(st64, sph)
    f64 = {k: np.asarray(want[k], dtype=np.float64) for k in WF[:4]}
    fin64 = np.isfinite(f64["opd"]) & np.isfinite(f64["pupil_x"])
    fin32 = np.isfinite(got["opd"]) & np.isfinite(got["pupil_x"])
    flip = (fin64 != fin32) | ((st64["i"] > 0) != (got["intensity"] > 0))
    assert np.mean(flip) <= 0.02, (name, int(flip.sum()))
    m = fin64 & fin32 & ~flip
    worst = 0.0
    for k in WF[:4]:
        dp, dD, do = part[k]
        tol = 3.0 * (dp * e["pos"] + dD * e["dir"] + do * e["opd"]) + U32 * np.abs(got[k])
        err = np.abs(got[k] - f64[k])
        bad = m & ~(err <= tol)
        assert not bad.any(), (name, k, int(bad.sum()), float(np.max(err[bad] / tol[bad])))
        worst = max(worst, float(np.max(err[m] / tol[m], initial=0.0)))
    ei = np.abs(got["intensity"] - st64["i"])
    assert np.all(ei[m] <= 3.0 * e["intensity"] + U32 * np.abs(st64["i"][m])), (name, float(np.max(ei[m])))
    print(f"{name}: fp32 against fp64, worst error / bound {worst:.3e} over {int(m.sum())} rays")


# ---- tiles round the grid-stride loop -----------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
def test_grid_stride_wraps(dtype):
    """A Double-Gauss pupil launch above SMs x 8 x 64 x BLOCK x RPT rays: the grid is at most 64x the resident CTAs and
    at most 8 CTAs of 256 threads fit on an SM, so tiles wrap round the grid-stride loop whatever the occupancy.  The
    first and last four tiles and a strided sample of >= 10^5 rays are checked against the long-double reference."""
    c, dtab = _case("dgauss_c2")
    rpt = _variant_rpt(dtab, dtype)
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    tile = BLOCK * rpt
    n = sms * 8 * 64 * tile + 5 * tile + 3
    aff = _affine(c)
    sph = dict(_spheres(c)[0], tilt=(0.05 * c.scale, -0.03 * c.scale))
    g = torch.Generator(device="cuda").manual_seed(3)
    r = torch.rand(n, generator=g, device="cuda", dtype=torch.float64).sqrt_()
    th = torch.rand(n, generator=g, device="cuda", dtype=torch.float64).mul_(2 * math.pi)
    Px = (r * torch.cos(th)).to(dtype)
    Py = (r * torch.sin(th)).to(dtype)
    del r, th
    src = ("pupil", (Px, Py, aff, None))
    sel = np.unique(np.concatenate([np.arange(4 * tile), np.arange(n - 4 * tile, n),
                                    np.linspace(4 * tile, n - 4 * tile, 100_003).astype(np.int64)]))
    sel_d = torch.from_numpy(sel).cuda()
    wf = _launch(dtab, dtype, n, src, wf=sph)["wf"]
    got = {k: v.index_select(0, sel_d).double().cpu().numpy() for k, v in wf.items()}
    del wf
    torch.cuda.empty_cache()
    fin = _launch(dtab, dtype, n, src, final=True)["fin"]
    st = {k: v.index_select(0, sel_d).double().cpu().numpy() for k, v in fin.items()}
    del fin
    px = Px.index_select(0, sel_d).double().cpu().numpy()
    py = Py.index_select(0, sel_d).double().cpu().numpy()
    del Px, Py
    torch.cuda.empty_cache()
    _, worst, _, _, _ = _check(got, st, px, py, sph, dtype, ("grid-stride", n))
    print(f"grid-stride {dtype}: {n} rays ({-(-n // tile)} tiles, grid <= {sms * 8 * 64}), worst error / bound {worst:.3e}")
