"""The fused spot-moment epilogue (``OlbTraceCall.moments``, the ``OLB_TF_MOMENTS`` block at the end of ``trace_kernel``)
on the GPU, in every flag combination, both precisions and every kernel variant that carries it.

The epilogue writes nothing per ray, so its reference is the SAME kernel's records: for each case one moments launch and
one records launch run on the same table, dtype and rays, and the 8 sums are rebuilt on the host from record row
``last - 1`` with ``math.fsum`` (correctly rounded).  ``_out_buffer`` pads the record stride to a vector multiple, so the
records launch runs the same rays-per-thread (RPT) instance as the moments launch for every ``n``.

Tolerances are derived, never picked:
* counts (``m[0]``, ``m[7]``) are integers below 2^53: exact;
* every other sum: the summation error bound ``(k + 8) u64 sum|terms|`` with ``k`` the longest addition chain of the
  kernel (per-thread partials, warp tree, one atomic per warp) -- see ``_chain``;
* local frame: the kernel's ``r.x`` is the local value itself, the host only sees it through the rounded global record;
  ``_local_slack`` bounds that difference per ray from the arithmetic of ``to_global``;
* fp32 against the fp64 reference: 3x the per-fixture achieved fp32 intercept error (``f32_achieved.json``), as the
  fp32 parity tests use it.
"""
from __future__ import annotations

import json
import math
import os

import numpy as np
import pytest
import torch

from tests._util import GOLDEN, Case

pytestmark = pytest.mark.gpu

BLOCK = 256                       # trace_kernel's block size (olb_trace.cu)
U64 = 2.0 ** -53
UNIT = {torch.float32: 2.0 ** -24, torch.float64: 2.0 ** -53}
FEAT_ROT = 1                      # olb_prep.h: FEAT_ROT; HINT_POLY_NEWTON
HINT_POLY_NEWTON = 1
CENTERS = ((0.0, 0.0), (41.5, -27.25))     # the origin, and a point far off every fixture's spot
MODES = ((False, False), (True, False), (False, True), (True, True))   # (global_xy, every_ray)
DTYPES = (torch.float32, torch.float64)

# fixture -> (RPT fp32, RPT fp64, inner `last` or None).  The RPT is trace_impl's rule: closed-form tables (planes /
# conics, rotated or not) 4 / 2, asphere-only Newton tables and tables with a non-radial aperture (FEAT_EXTRA) 2 / 1,
# polynomial-family Newton tables 1 / 1, and every phase / grating / grid-sag / polygon superset one ray per thread.
# tilted_fold's rectangular aperture puts it in the general kernel; "tilted_fold:open" is its table without apertures,
# which reaches the closed-form FEAT_ROT instance.  The inner `last` ends on a rotated surface
# (tilted_fold, polygon_nested_tilted), on hubble_c4's obscured primary, and on the dgauss_nan row whose NaN rays still
# carry i > 0 (the m[7] path through the closed form).
MATRIX = {
    "dgauss_c2": (4, 2, None),
    "tilted_fold": (2, 1, 4),
    "tilted_fold:open": (4, 2, 4),
    "hubble_c4": (4, 2, 3),
    "dgauss_nan": (4, 2, 8),
    "aspheric_singlet": (2, 1, None),
    "zernike_fringe": (1, 1, None),
    "cheb_biconic_toroidal": (1, 1, None),
    "phase/phase_doe_achromat": (1, 1, None),
    "grating/grating_high_orders": (1, 1, None),
    "grid_sag/grid_nan_patterns": (1, 1, None),
    "polygon_aperture/polygon_nan_rays": (1, 1, None),
    "polygon_aperture/polygon_nested_tilted": (1, 1, 4),
}
CASES = [(name, last) for name, (_, _, inner) in MATRIX.items() for last in ((None,) if inner is None else (None, inner))]
CASE_IDS = [f"{n}-last{l}" if l else n for n, l in CASES]


def _sizes(name, dtype):
    """1, 3, 5, a warp-multiple +- 1, BLOCK*RPT +- 1 (tile boundary of this instance) and a ragged 4099."""
    rpt = MATRIX[name][0 if dtype == torch.float32 else 1]
    return sorted({1, 3, 5, 255, 257, BLOCK * rpt - 1, BLOCK * rpt + 1, 4099})


_TABLES: dict = {}


def _case(name):
    from optiland_b200.trace import DeviceTable

    if name not in _TABLES:
        base, _, variant = name.partition(":")
        c = Case(base)
        if variant == "open":
            for s in c.table.surfaces:
                s.aperture = None
        _TABLES[name] = (c, DeviceTable(c.table))
    return _TABLES[name]


def _rpt(dtab, dtype):
    """trace_impl's rays-per-thread rule (olb_trace.cu), from the uploaded table's feature bits and hints."""
    closed = (dtab.features & ~FEAT_ROT) == 0
    poly = (dtab.c.hints & HINT_POLY_NEWTON) != 0
    if dtype == torch.float32:
        return 4 if closed else (1 if poly else 2)
    return 2 if closed else 1


def _variant_rpt(dtab, dtype):
    """The RPT of the kernel instance actually launched: the phase / grating / grid / polygon supersets run 1."""
    supersets = (1 << 5) | (1 << 6) | (1 << 8) | (1 << 9)
    return 1 if dtab.features & supersets else _rpt(dtab, dtype)


def _chain(n, rpt):
    """Longest chain of fp64 additions from one ray's term to a moment: the thread's partial sum (RPT rays per tile,
    grid-stride over the tiles; the grid is min(tiles, SMs x resident CTAs x 64) >= min(tiles, 64 x SMs)), the 5-level
    warp tree, then one atomicAdd per warp of the grid (at most BLOCK/32 per tile) in any order."""
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    tiles = -(-n // (BLOCK * rpt))
    grid_min = min(tiles, 64 * sms)
    return rpt * -(-tiles // grid_min) + 5 + (BLOCK // 32) * tiles


def _local_slack(g, s, u):
    """Per-ray bound of |kernel local x - fp64 host transform of the rounded global record| (and the same for y).

    The kernel's global record is g = fl(R' r + t') with R', t' the table's R, t rounded to T (one u each) and three
    nested FMAs (to_global, 3 u): |g - (R r + t)|_j <= 5 u (sum_i |R_ji| |r_i| + |t_j|) <= 5 u (|r|_1 + |t|_1).
    The host forms R^T (g - t), so it sees r + R^T delta: per component <= sqrt(3) |delta|_inf (rows of R are unit
    vectors), and |r|_1 <= sqrt(3) (|g|_1 + |t|_1).  Altogether 5 sqrt(3) (sqrt(3) + 1) u (|g|_1 + |t|_1) < 24 u (...);
    32 also covers the host's own fp64 rounding (4 operations of u64 <= u each)."""
    t1 = float(np.sum(np.abs(np.asarray(s.t, dtype=np.float64))))
    return 32.0 * u * (np.abs(g[0]) + np.abs(g[1]) + np.abs(g[2]) + t1)


def _host_terms(c, rec, last, center, glob, every, dtype):
    """The per-ray terms the kernel sums (olb_trace.cu, OLB_TF_MOMENTS): dx = float64(x) - cx etc., the mask
    i > 0 && finite / every ray, and m[7] = i > 0 but not finite; plus the per-moment slack of the local frame."""
    row = last - 1
    g = [rec[k][row].double().cpu().numpy() for k in ("x", "y", "z")]
    ii = rec["intensity"][row].double().cpu().numpy()
    oo = rec["opd"][row].double().cpu().numpy()
    if glob:
        x, y = g[0], g[1]
        e = np.zeros_like(x)
    else:
        s = c.table.surfaces[last - 1]
        tx, ty, tz = (float(v) for v in s.t)
        dx, dy, dz = g[0] - tx, g[1] - ty, g[2] - tz
        if s.rotated:       # local = R^T (global - t), as spot.py::_materialize
            R = s.R
            x = R[0, 0] * dx + R[1, 0] * dy + R[2, 0] * dz
            y = R[0, 1] * dx + R[1, 1] * dy + R[2, 1] * dz
        else:
            x, y = dx, dy
        e = _local_slack(g, s, UNIT[dtype])
    dx, dy = x - center[0], y - center[1]
    finite = np.isfinite(dx) & np.isfinite(dy)
    sel = np.ones(dx.shape, bool) if every else (ii > 0) & finite
    m7 = 0 if every else int(np.count_nonzero(~sel & (ii > 0)))
    dx, dy, e, ii, oo = dx[sel], dy[sel], e[sel], ii[sel], oo[sel]
    terms = [dx, dy, dx * dx + dy * dy, ii, oo, oo * oo]
    with np.errstate(invalid="ignore"):
        ax, ay = np.abs(dx), np.abs(dy)
        slack = [float(np.sum(e)), float(np.sum(e)), float(np.sum(2.0 * (ax + ay) * e + 2.0 * e * e)), 0.0, 0.0, 0.0]
    return int(np.count_nonzero(sel)), m7, terms, slack


def _assert_sums(got, want, k, ctx):
    """m[0], m[7] exact; m[1..6] within (k + 8) u64 sum|terms| (+ the local-frame slack) of the correctly rounded
    sum.  The 8 beyond the chain cover the term itself: dx*dx + dy*dy may be contracted to an FMA in the kernel."""
    cnt, m7, terms, slack = want
    got = [float(v) for v in got.cpu()]
    assert got[0] == cnt, (ctx, "count", got[0], cnt)
    assert got[7] == m7, (ctx, "m7", got[7], m7)
    for q, (t, sl) in enumerate(zip(terms, slack), start=1):
        if not np.all(np.isfinite(t)):
            # a NaN ray in the sums (every-ray mode): the kernel's sum is NaN as well, as the reference's be.mean
            if np.any(np.isnan(t)):
                assert math.isnan(got[q]), (ctx, q, got[q])
            else:
                assert not math.isfinite(got[q]), (ctx, q, got[q])
            continue
        ref = math.fsum(t.tolist())
        tol = (k + 8) * U64 * math.fsum(np.abs(t).tolist()) + sl
        assert abs(got[q] - ref) <= tol, (ctx, q, got[q], ref, tol)


def _rays(c, idx, dtype):
    from optiland_b200.trace import RealRays

    r = {k: np.ascontiguousarray(v[idx]) for k, v in c.rays.items()}
    return RealRays(r["x"], r["y"], r["z"], r["L"], r["M"], r["N"], r["i"], r["w"], dtype=dtype)


def _launch_scalars(c):
    return {k[9:]: float(c.z[k]) for k in c.z.files if k.startswith("x_launch_")}


def _forms(c, dtab, idx, dtype, last):
    """(tag, moments(center, glob, every), records) for the ray-array form and, where the fixture has pupil samples
    and launch scalars, the pupil-launch form; the moment launches run before the records launch on the same rays."""
    from optiland_b200.launch import pupil_affine
    from optiland_b200.trace import trace_device, trace_moments_device, trace_pupil_device

    n = idx.size
    rays = _rays(c, idx, dtype)
    x_in = rays.x.clone()

    def mom_rays(center, glob, every):
        return trace_moments_device(dtab, n, dtype, rays=rays, center=center, last=last, global_xy=glob,
                                    every_ray=every)

    got = {(cen, m): mom_rays(cen, *m) for cen in CENTERS for m in MODES}
    assert torch.equal(rays.x, x_in)            # the launch arrays are only read
    rec = trace_device(dtab, rays, 0, last, record=True)
    out = [("rays", got, rec)]
    if "x_Px" in c.z.files and _launch_scalars(c):
        aff = pupil_affine(_launch_scalars(c))
        Px = torch.from_numpy(np.ascontiguousarray(c.extra("Px")[idx])).to("cuda", dtype)
        Py = torch.from_numpy(np.ascontiguousarray(c.extra("Py")[idx])).to("cuda", dtype)
        got_p = {(cen, m): trace_moments_device(dtab, n, dtype, pupil=(Px, Py, aff), center=cen, last=last,
                                                global_xy=m[0], every_ray=m[1]) for cen in CENTERS for m in MODES}
        _, rec_p = trace_pupil_device(dtab, Px, Py, aff, 0, last)
        out.append(("pupil", got_p, rec_p))
    return out


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("name,last", CASES, ids=CASE_IDS)
def test_moments_equal_exact_sums_of_the_records(name, last, dtype):
    """Every mode (masked local / masked global / every-ray local / every-ray global) x center x tail size: the
    epilogue's 8 sums == the correctly rounded sums of the same kernel's records, within the summation bound."""
    c, dtab = _case(name)
    rpt = _variant_rpt(dtab, dtype)
    assert rpt == MATRIX[name][0 if dtype == torch.float32 else 1], "the fixture no longer reaches its kernel variant"
    last = c.table.num_surfaces if last is None else last
    if last < c.table.num_surfaces:
        assert c.table.surfaces[last - 1].kind != 0     # a traced surface: its local frame is the kernel's r.x
    for n in _sizes(name, dtype):
        idx = np.random.default_rng(n).integers(0, c.n, size=n)
        k = _chain(n, rpt)
        for form, got, rec in _forms(c, dtab, idx, dtype, last):
            for (cen, (glob, every)), m in got.items():
                want = _host_terms(c, rec, last, cen, glob, every, dtype)
                _assert_sums(m, want, k, (form, n, cen, "global" if glob else "local", "all" if every else "masked"))


# the polygon fixtures have no achieved-error file: their suite bounds fp32 intercepts by this fraction of the system's
# scale (test_polygon_apertures.F32_POS) and leaves polygon_nan_rays' ill-conditioned grazing rays out of fp32 checks
POLYGON_F32_POS = 4e-6
F32_CASES = [(name, last) for name, last in CASES if "nan_rays" not in name]


def _f32_pos_bound(c, name):
    """Per-ray bound (mm) of the fp32 kernel's intercepts against fp64: 3x the error the fp32 arithmetic achieves on
    this fixture (f32_achieved.json), or the polygon suite's bound."""
    base = name.partition(":")[0]
    if base.startswith("polygon_aperture/"):
        return POLYGON_F32_POS * c.scale
    sub, case = os.path.split(base)
    with open(os.path.join(GOLDEN, sub, "f32_achieved.json")) as f:
        return 3.0 * json.load(f)["cases"][case]["pos"]


def _fp64_rows(c, idx, last):
    """The fp64 intercepts of row last - 1: the NumPy oracle for the core surface families; for the phase / grating /
    grid-sag / polygon fixtures (outside trace_oracle) the reference's own fp64 records of the same rays."""
    row = last - 1
    if "/" in c.name:
        return c.rec["x"][row][idx], c.rec["y"][row][idx], c.rec["intensity"][row][idx]
    from oracle import trace_oracle as O

    _, orec, _ = O.trace(c.table, {k: v[idx] for k, v in c.rays.items()}, 0, last)
    return orec["x"][row], orec["y"][row], orec["intensity"][row]


@pytest.mark.parametrize("name,last", F32_CASES, ids=[f"{n}-last{l}" if l else n for n, l in F32_CASES])
def test_f32_moments_against_the_fp64_reference(name, last):
    """fp32 centroid and RMS radius (global frame, masked and every-ray) against fp64: the centroid within the per-ray
    fp32 intercept bound e (a mean of per-ray errors <= e), the RMS radius about the centroid within sqrt(2) e (|rms_a - rms_b| <= the RMS of the per-ray 2-D displacement differences, triangle inequality)."""
    from optiland_b200.trace import trace_device, trace_moments_device

    c, dtab = _case(name)
    last = c.table.num_surfaces if last is None else last
    e = _f32_pos_bound(c, name)
    n = 4099
    idx = np.random.default_rng(7).integers(0, c.n, size=n)
    x, y, i = _fp64_rows(c, idx, last)
    rays = _rays(c, idx, torch.float32)
    rec = trace_device(dtab, _rays(c, idx, torch.float32), 0, last, record=True)
    gx = rec["x"][last - 1].double().cpu().numpy()
    gy = rec["y"][last - 1].double().cpu().numpy()
    gi = rec["intensity"][last - 1].double().cpu().numpy()
    fin, fin32 = np.isfinite(x) & np.isfinite(y), np.isfinite(gx) & np.isfinite(gy)
    if not (np.array_equal(fin, fin32) and np.array_equal(i > 0, gi > 0)):
        # fp32 may turn a grazing ray into a miss (and back): the parity tests allow 2 % such rays; the statistics of
        # two different ray sets are not comparable
        assert np.mean((fin != fin32) | ((i > 0) != (gi > 0))) <= 0.02
        return
    for every in (False, True):
        sel = np.ones(n, bool) if every else (i > 0) & fin
        m = trace_moments_device(dtab, n, torch.float32, rays=rays, last=last, global_xy=True, every_ray=every)
        m = [float(v) for v in m.cpu()]
        assert m[0] == np.count_nonzero(sel)
        if m[0] == 0:
            continue
        xs, ys = x[sel], y[sel]
        if not (np.all(np.isfinite(xs)) and np.all(np.isfinite(ys))):
            assert math.isnan(m[1]) and math.isnan(m[3])
            continue
        cx, cy = xs.mean(), ys.mean()
        assert abs(m[1] / m[0] - cx) <= e and abs(m[2] / m[0] - cy) <= e, (every, m[1] / m[0], cx, m[2] / m[0], cy)
        # second moments about the fp64 centroid: no cancellation against the offset of the spot
        mc = [float(v) for v in trace_moments_device(dtab, n, torch.float32, rays=rays, center=(cx, cy), last=last,
                                                     global_xy=True, every_ray=every).cpu()]
        rms = math.sqrt(max(mc[3] / mc[0] - (mc[1] / mc[0]) ** 2 - (mc[2] / mc[0]) ** 2, 0.0))
        ref = math.sqrt(np.mean((xs - cx) ** 2 + (ys - cy) ** 2))
        assert abs(rms - ref) <= math.sqrt(2.0) * e, (every, rms, ref)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
def test_ten_million_ray_pupil_launch(dtype):
    """10^7 rays of the Double-Gauss pupil (as test_full_size_properties_double_gauss), the grid oversubscribed 64x:
    the sums still match the records to the summation bound, which at this size is ~1e-11 of sum|terms| -- a single
    lost or extra ray (1e-7 of it) would be 4 orders of magnitude outside."""
    from optiland_b200.launch import pupil_affine
    from optiland_b200.trace import trace_moments_device, trace_pupil_device

    c, dtab = _case("dgauss_c2")
    aff = pupil_affine(_launch_scalars(c))
    n = 10_000_000
    g = torch.Generator(device="cuda").manual_seed(0)
    r = torch.rand(n, generator=g, device="cuda", dtype=torch.float64).sqrt()
    th = 2 * np.pi * torch.rand(n, generator=g, device="cuda", dtype=torch.float64)
    Px, Py = (r * torch.cos(th)).to(dtype), (r * torch.sin(th)).to(dtype)
    del r, th
    last = c.table.num_surfaces
    modes = ((False, False), (True, True))
    cen = CENTERS[1]
    got = {m: trace_moments_device(dtab, n, dtype, pupil=(Px, Py, aff), center=cen, global_xy=m[0], every_ray=m[1])
           for m in modes}
    _, rec = trace_pupil_device(dtab, Px, Py, aff, 0, last)
    k = _chain(n, _variant_rpt(dtab, dtype))
    for m in modes:
        _assert_sums(got[m], _host_terms(c, rec, last, cen, m[0], m[1], dtype), k, ("1e7", m))


# ---- the two consumers, against the reference's definitions ----------------------------------------------------------

class _RaysEngine:
    """The engine's ``spot_moments`` contract (plugin.CudaEngine) on a fixed ray batch instead of a pupil launch, so the
    consumers in spot.py can be driven by the real kernel on golden rays; records the launches it made."""

    def __init__(self, dtab, rays):
        self.dtab, self.rays, self.calls = dtab, rays, []

    def spot_moments(self, table, Px, Py, affine, center=(0.0, 0.0), last=None, global_xy=False, every_ray=False):
        from optiland_b200.trace import trace_moments_device

        self.calls.append(("moments", last, global_xy, every_ray))
        m = trace_moments_device(self.dtab, len(self.rays), self.rays.dtype, rays=self.rays, center=center, last=last,
                                 global_xy=global_xy, every_ray=every_ray)
        return [float(v) for v in m.cpu()]


def _records(c, dtab, idx, dtype, last=None):
    from optiland_b200.trace import trace_device

    last = c.table.num_surfaces if last is None else last
    rec = trace_device(dtab, _rays(c, idx, dtype), 0, last, record=True)
    return {k: v[last - 1].double().cpu().numpy() for k, v in rec.items()}


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("name", ["grating/grating_high_orders", "polygon_aperture/polygon_nan_rays", "hubble_c4"])
def test_lazy_spot_data_follows_the_reference_mean(name, dtype):
    """LazySpotData.centroid / rms_about (SpotDiagram, masked local frame) == the reference's be.mean over the i > 0
    rays: NaN as soon as one kept ray is not finite (m[7] > 0: grating_high_orders' evanescent orders), the plain mean
    otherwise (polygon_nan_rays' NaN rays are vignetted, i == 0, so they drop out)."""
    from optiland_b200.spot import LazySpotData

    c, dtab = _case(name)
    idx = np.arange(c.n)
    eng = _RaysEngine(dtab, _rays(c, idx, dtype))
    sd = LazySpotData(eng, None, c.table, None, None, None, "local")
    r = _records(c, dtab, idx, dtype)
    s = c.table.surfaces[-1]
    assert not s.rotated
    keep = r["intensity"] > 0
    x, y = r["x"][keep] - float(s.t[0]), r["y"][keep] - float(s.t[1])
    cx, cy = sd.centroid()
    if not (np.all(np.isfinite(x)) and np.all(np.isfinite(y))):
        assert sd.moments()[7] > 0
        assert math.isnan(cx) and math.isnan(cy) and math.isnan(sd.rms_about(0.0, 0.0))
        return
    # centroid: the mean of n values, each within the local-frame slack of the kernel's, summed within (k + 8) u64
    n = x.size
    e = float(np.max(_local_slack([r["x"][keep], r["y"][keep], r["z"][keep]], s, UNIT[dtype])))
    k = _chain(len(idx), _variant_rpt(dtab, dtype))
    assert abs(cx - x.mean()) <= e + (k + 8) * U64 * np.abs(x).mean()
    assert abs(cy - y.mean()) <= e + (k + 8) * U64 * np.abs(y).mean()
    ref = math.sqrt(np.mean((x - cx) ** 2 + (y - cy) ** 2))
    assert sd.rms_about(cx, cy) == pytest.approx(ref, abs=2 * e + (k + 8) * U64 * ref)


class _Stub:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def _operand(monkeypatch, c, dtab, rays, surface_number):
    """spot.rms_spot_size (the RayOperand.rms_spot_size consumer) with its launch inputs replaced by a fixed batch."""
    from optiland_b200 import spot

    eng = _RaysEngine(dtab, rays)
    monkeypatch.setattr(spot, "_fused_inputs", lambda *a, **k: ((c.table, None, None, None), None))
    P = _Stub(_state={"engine": eng})
    optic = _Stub(surfaces=_Stub(num_surfaces=c.table.num_surfaces))
    be = _Stub(array=lambda v: np.asarray(v, dtype=np.float64))
    out = float(spot.rms_spot_size(P, None, be, optic, surface_number, 0.0, 0.0, len(rays), 0.55, object()))
    assert eng.calls and all(call[2:] == (True, True) for call in eng.calls)     # GLOBAL | ALL launches only
    return out


def _reference_rms_spot_size(x, y):
    """optiland/optimization/operand/ray.py rms_spot_size for one wavelength: be.mean over EVERY ray of the row."""
    xc, yc = np.mean(x), np.mean(y)
    return float(np.sqrt(np.mean((x - xc) ** 2 + (y - yc) ** 2)))


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
def test_operand_counts_vignetted_rays_and_propagates_nan(monkeypatch, dtype):
    """rms_spot_size from every-ray moments: hubble_c4's obscured rays (i == 0) are counted, as in the reference's
    unmasked be.mean (and the value differs from the masked one); one NaN ray among finite ones makes it NaN."""
    c, dtab = _case("hubble_c4")
    idx = np.arange(c.n)
    r = _records(c, dtab, idx, dtype)
    assert np.count_nonzero(r["intensity"] == 0) > 0
    got = _operand(monkeypatch, c, dtab, _rays(c, idx, dtype), -1)
    want = _reference_rms_spot_size(r["x"], r["y"])
    masked = _reference_rms_spot_size(r["x"][r["intensity"] > 0], r["y"][r["intensity"] > 0])
    # second moments about the kernel's own centroid, summed within (k + 8) u64 (both sides read the same records)
    k = _chain(len(idx), _variant_rpt(dtab, dtype))
    tol = 2 * (k + 8) * U64 * want
    assert got == pytest.approx(want, abs=tol) and abs(masked - want) > 1e3 * tol

    cn, dn = _case("dgauss_nan")
    rn = _records(cn, dn, np.arange(cn.n), dtype)
    bad = np.flatnonzero(np.isnan(rn["x"]))
    good = np.flatnonzero(np.isfinite(rn["x"]) & np.isfinite(rn["y"]))
    assert bad.size and good.size
    one = np.concatenate([good, bad[:1]])
    assert math.isnan(_operand(monkeypatch, cn, dn, _rays(cn, one, dtype), -1))
    assert math.isfinite(_operand(monkeypatch, cn, dn, _rays(cn, good, dtype), -1))


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
def test_global_and_local_frames_differ_on_the_tilted_fold(dtype):
    """tilted_fold, traced to its tilted, decentred third surface: the global and local centroids are different
    points, and each equals its own host transform of the records (the equality itself is the matrix test's)."""
    from optiland_b200.trace import trace_moments_device

    c, dtab = _case("tilted_fold")
    last = 4
    s = c.table.surfaces[last - 1]
    assert s.rotated
    idx = np.arange(c.n)
    rays = _rays(c, idx, dtype)
    mg = trace_moments_device(dtab, c.n, dtype, rays=rays, last=last, global_xy=True)
    ml = trace_moments_device(dtab, c.n, dtype, rays=rays, last=last)
    r = _records(c, dtab, idx, dtype, last)
    d = np.stack([r["x"] - s.t[0], r["y"] - s.t[1], r["z"] - s.t[2]])
    loc = s.R.T @ d
    e = float(np.max(_local_slack([r["x"], r["y"], r["z"]], s, UNIT[dtype])))
    k = _chain(c.n, _variant_rpt(dtab, dtype))
    for m, (x, y), slack in ((mg, (r["x"], r["y"]), 0.0), (ml, (loc[0], loc[1]), e)):
        m = [float(v) for v in m.cpu()]
        assert m[0] == c.n
        assert abs(m[1] / m[0] - x.mean()) <= slack + (k + 8) * U64 * np.abs(x).mean()
        assert abs(m[2] / m[0] - y.mean()) <= slack + (k + 8) * U64 * np.abs(y).mean()
    gap = math.hypot(float(mg[1] - ml[1]), float(mg[2] - ml[2])) / c.n
    assert gap > 100.0 * (e + (k + 8) * U64 * c.scale)


# ---- live Optiland at float32 precision on the CUDA engine -----------------------------------------------------------

@pytest.fixture
def plugin_f32():
    from oracle.ref_import import import_reference, reference_available

    if not reference_available():
        pytest.skip("reference not present on this box")
    import_reference()
    import optiland.backend as be

    from optiland_b200 import _lib
    from optiland_b200 import plugin as P

    be.set_backend("torch")
    be.set_precision("float32")
    be.grad_mode.disable()
    be.set_device("cuda")
    eng = P.CudaEngine()
    launches0 = _lib.load().olb_launch_count()
    P.install(engine=eng)
    P.stats(reset=True)
    yield P, eng, be
    assert not eng.calls or _lib.load().olb_launch_count() > launches0
    be.set_device("cpu")
    be.set_precision("float64")
    P.uninstall()
    be.set_backend("numpy")


def _f32_pos(name):
    with open(os.path.join(GOLDEN, "f32_achieved.json")) as f:
        return json.load(f)["cases"][name]["pos"]


def test_live_spot_diagram_at_float32(plugin_f32):
    """SpotDiagram(CookeTriplet) at be.set_precision("float32"): rms_spot_radius / centroid from fp32 moment launches
    against the NumPy reference in fp64, both reference strategies.  Bounds from the achieved fp32 intercept error of
    the Cooke triplet (cooke_c1) e: centroid 3 e, RMS radius 3 sqrt(2) e (see test_f32_moments_against_the_fp64_reference);
    the chief-ray reference point is itself an fp32 intercept, which adds at most 3 e to the radius."""
    P, eng, be = plugin_f32
    from optiland.analysis import SpotDiagram
    from optiland.samples.objectives import CookeTriplet

    e = 3.0 * _f32_pos("cooke_c1")
    for reference in ("chief_ray", "centroid"):
        be.set_backend("numpy")
        be.set_precision("float64")
        ref = SpotDiagram(CookeTriplet(), reference=reference)
        want = np.array(ref.rms_spot_radius(), dtype=np.float64)
        want_c = np.array(ref.centroid(), dtype=np.float64)
        be.set_backend("torch")
        be.set_precision("float32")
        n0 = len(eng.calls)
        spot = SpotDiagram(CookeTriplet(), reference=reference)
        got = np.array([[float(v) for v in row] for row in spot.rms_spot_radius()])
        got_c = np.array([[float(v) for v in cc] for cc in spot.centroid()])
        new = eng.calls[n0:]
        assert [cc[0] for cc in new].count("moments") >= 9 and not any(cc[0] == "pupil" and cc[2] > 1 for cc in new), new
        np.testing.assert_allclose(got_c, want_c, rtol=0, atol=e)
        np.testing.assert_allclose(got, want, rtol=0, atol=math.sqrt(2.0) * e + (e if reference == "chief_ray" else 0.0))
    assert not any("spot moments" in k for k in P.stats()), P.stats()


@pytest.mark.parametrize("surface_number,wavelength", [(-1, 0.55), (-1, "all"), (2, 0.55), (2, "all")])
def test_live_rms_spot_size_operand_at_float32(plugin_f32, surface_number, wavelength):
    """RayOperand.rms_spot_size on the Hubble telescope at float32 precision, image and primary mirror, one wavelength
    and "all": served by every-ray global moment launches, within 3 sqrt(2) e of the fp64 NumPy reference (e: the
    achieved fp32 intercept error of hubble_c4)."""
    P, eng, be = plugin_f32
    from optiland.optimization.operand.ray import RayOperand
    from optiland.samples.telescopes import HubbleTelescope

    args = dict(surface_number=surface_number, Hx=0.0, Hy=1.0, num_rays=8, wavelength=wavelength)
    be.set_backend("numpy")
    be.set_precision("float64")
    want = float(RayOperand.rms_spot_size(HubbleTelescope(), distribution="hexapolar", **args))
    be.set_backend("torch")
    be.set_precision("float32")
    n0 = len(eng.calls)
    got = float(RayOperand.rms_spot_size(HubbleTelescope(), distribution="hexapolar", **args))
    assert all(cc[0] == "moments" for cc in eng.calls[n0:]) and len(eng.calls) > n0, eng.calls[n0:]
    assert abs(got - want) <= 3.0 * math.sqrt(2.0) * _f32_pos("hubble_c4"), (got, want)


# ---- SurfaceGroup.spot_moments: the RMS radius of a small spot far from `center` ------------------------------------

def test_spot_moments_rms_of_a_micrometre_spot_20mm_off_axis():
    """A ~1 um spot at 19.7 mm image height (the Double-Gauss at Hy = 0.8 with the pupil stopped down to 5 %), 10^6 rays,
    fp64.  moments_to_spot's one-pass variance m3/n - mx^2 - my^2 about (0, 0) subtracts two ~390 mm^2 numbers to get
    ~1e-6 mm^2: the rounding of the sums (u64 x 390 mm^2 per addition) is amplified ~4e8-fold.  Measured on an
    H100 80GB HBM3 (700 W power limit): relative error of rms_centroid 1.6e-6 in one pass.  SurfaceGroup.spot_moments takes the second moments
    about the first pass's centroid instead; it must then agree with the two-pass fsum of the records to 1e-9."""
    from optiland_b200.launch import pupil_affine
    from optiland_b200.trace import SurfaceGroup, moments_to_spot, trace_moments_device, trace_pupil_device

    c = Case("dgauss_c2")
    sg = SurfaceGroup(c.table)
    aff = pupil_affine(dict(_launch_scalars(c), Hy=0.8))
    n = 1_000_000
    g = torch.Generator(device="cuda").manual_seed(5)
    r = 0.05 * torch.rand(n, generator=g, device="cuda", dtype=torch.float64).sqrt()
    th = 2 * np.pi * torch.rand(n, generator=g, device="cuda", dtype=torch.float64)
    Px, Py = r * torch.cos(th), r * torch.sin(th)
    _, rec = trace_pupil_device(sg.device_table, Px, Py, aff, 0, c.table.num_surfaces)
    x, y = rec["x"][-1].cpu().numpy(), rec["y"][-1].cpu().numpy()
    assert np.all(rec["intensity"][-1].cpu().numpy() > 0) and np.all(np.isfinite(x) & np.isfinite(y))
    cx, cy = math.fsum(x.tolist()) / n, math.fsum(y.tolist()) / n
    ref = math.sqrt(math.fsum(((x - cx) ** 2 + (y - cy) ** 2).tolist()) / n)
    assert 19.0 < cy < 21.0 and 0.5e-3 < ref < 2e-3
    one_pass = moments_to_spot(trace_moments_device(sg.device_table, n, torch.float64, pupil=(Px, Py, aff)))
    print(f"one-pass rms_centroid relative error: {abs(one_pass['rms_centroid'] - ref) / ref:.3e}")
    got = sg.spot_moments(pupil=(Px, Py, aff))
    assert got["count"] == n
    assert got["centroid"][1] == pytest.approx(cy, rel=1e-12)
    assert abs(got["rms_centroid"] - ref) <= 1e-9 * ref, (got["rms_centroid"], ref, one_pass["rms_centroid"])
    assert got["rms_center"] == pytest.approx(math.hypot(cx, cy), rel=1e-6)
