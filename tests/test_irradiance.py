"""Incoherent irradiance binning (olb_irradiance_*, optiland_b200/irradiance.py): the kernel's per-ray arithmetic against
np.histogram2d on adversarial inputs, the ABI's argument checks, and the plugin's ``IncoherentIrradiance`` wrapper
against the reference's own body -- live on the CPU through the host build of the arithmetic, and on the GPU through
the kernel."""
import ctypes as C
import io
import os
import re
import subprocess
import sys
import tempfile
from contextlib import redirect_stdout

import numpy as np
import pytest

from oracle.ref_import import reference_available
from optiland_b200 import _lib

needs_ref = pytest.mark.skipif(not reference_available(), reason="reference not staged under oracle/_ref (build())")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- adversarial samples -----------------------------------------------------------------------------------------------

def _edges(kind):
    if kind == "linspace":
        return np.linspace(-2.5, 2.5, 8 + 1), np.linspace(-1.0, 3.0, 5 + 1)
    return np.arange(-2.5, 2.5 + 0.5 * 0.3, 0.3), np.arange(-1.0, 3.0 + 0.5 * 0.7, 0.7)   # px_size edges


def _samples(xe, ye, dtype, seed=0):
    """Points on every edge of each axis, one ulp (of the sample type) either side, NaN / +-inf coordinates, random points
    inside and outside, and powers that are positive, zero, negative and NaN."""
    rng = np.random.default_rng(seed)
    axis_vals = []
    for e in (xe, ye):
        v = e.astype(dtype)
        vals = np.concatenate([v, np.nextafter(v, dtype(np.inf)), np.nextafter(v, dtype(-np.inf)),
                               np.array([np.nan, np.inf, -np.inf], dtype=dtype),
                               rng.uniform(e[0] - 0.5, e[-1] + 0.5, 64).astype(dtype)])
        axis_vals.append(vals)
    X, Y = np.meshgrid(axis_vals[0], axis_vals[1], indexing="ij")
    x, y = X.ravel().astype(dtype), Y.ravel().astype(dtype)
    p = rng.uniform(0.1, 2.0, x.size).astype(dtype)
    p[::7] = 0
    p[3::11] = -1.0
    p[5::13] = np.nan
    return x, y, p


def _reference_bins(x, y, p, xe, ye):
    """np.histogram2d's bin of every ray (searchsorted side='right' - 1, the last edge inside), -1 when dropped."""
    out = np.full(x.size, -1, dtype=np.int64)
    idx = []
    for v, e in ((x, xe), (y, ye)):
        vd = v.astype(np.float64)
        k = np.searchsorted(e, vd, side="right") - 1
        k[vd == e[-1]] = len(e) - 2
        ok = (vd >= e[0]) & (vd <= e[-1])
        idx.append((k, ok))
    keep = (p > 0) & idx[0][1] & idx[1][1]
    out[keep] = idx[0][0][keep] * (len(ye) - 1) + idx[1][0][keep]
    return out


def _histogram2d(x, y, p, xe, ye):
    keep = p > 0
    return np.histogram2d(x[keep], y[keep], bins=[xe, ye], weights=p[keep])[0]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("kind", ["linspace", "arange"])
def test_host_arithmetic_matches_histogram2d(dtype, kind):
    from oracle.hostcheck_irradiance import bin_rays

    xe, ye = _edges(kind)
    x, y, p = _samples(xe, ye, dtype)
    bins, hist = bin_rays(x, y, p, xe, ye)
    assert np.array_equal(bins, _reference_bins(x, y, p, xe, ye))
    want = _histogram2d(x, y, p, xe, ye)
    assert hist.shape == want.shape
    np.testing.assert_allclose(hist, want, rtol=1e-12, atol=0)
    assert (bins >= 0).sum() > 100 and (bins < 0).sum() > 100


def test_host_arithmetic_translation_in_ray_precision():
    """An unrotated frame subtracts its origin in the rays' own precision, as the reference's translate does."""
    from oracle.hostcheck_irradiance import bin_rays

    xe, ye = _edges("linspace")
    x, y, p = _samples(xe, ye, np.float32, seed=3)
    t = np.array([0.1, -0.37, 5.0])
    xs, ys = (x + np.float32(t[0])).astype(np.float32), (y + np.float32(t[1])).astype(np.float32)
    bins, hist = bin_rays(xs, ys, p, xe, ye, frame=("translate", t))
    xl, yl = xs - np.float32(t[0]), ys - np.float32(t[1])
    assert np.array_equal(bins, _reference_bins(xl, yl, p, xe, ye))
    np.testing.assert_allclose(hist, _histogram2d(xl, yl, p, xe, ye), rtol=1e-12, atol=0)


# ---- the C ABI's checks (all before any device call) --------------------------------------------------------------------

def _call(**over):
    buf = np.zeros(16)
    xe = over.pop("xe", np.linspace(0, 1, 5))
    ye = over.pop("ye", np.linspace(0, 1, 4))
    c = _lib.OlbIrradiance(x=buf.ctypes.data, y=buf.ctypes.data, z=buf.ctypes.data, i=buf.ctypes.data, n_rays=16,
                           frame=0, nx=len(xe) - 1, ny=len(ye) - 1, x_edges=xe.ctypes.data, y_edges=ye.ctypes.data,
                           edges=buf.ctypes.data, hist=buf.ctypes.data)
    for k, v in over.items():
        setattr(c, k, v)
    rc = _lib.load().olb_irradiance_f64(C.byref(c), None)
    return rc, _lib.last_error()


def test_struct_size():
    assert C.sizeof(_lib.OlbIrradiance) == 184


@pytest.mark.parametrize("case,msg", [
    (dict(x=None), "NULL array"), (dict(hist=None), "NULL array"), (dict(edges=None), "NULL array"),
    (dict(frame=1, z=None), "NULL array"), (dict(frame=7), "frame"), (dict(nx=0), "nx and ny"),
    (dict(ny=-1), "nx and ny"), (dict(n_rays=-1), "n_rays"),
    (dict(xe=np.array([0.0, 1.0, 1.0, 2.0])), "x_edges"), (dict(xe=np.array([0.0, np.nan, 2.0])), "x_edges"),
    (dict(ye=np.array([0.0, 2.0, 1.0])), "y_edges"), (dict(ye=np.array([-np.inf, 0.0])), "y_edges"),
    (dict(path=3), "path"), (dict(path=-1), "path"),
    (dict(path=1, xe=np.linspace(0, 1, 200), ye=np.linspace(0, 1, 200)), "OLB_IRR_PATH_SHARED"),
])
def test_abi_rejects_bad_arguments(case, msg):
    rc, err = _call(**case)
    assert rc == -1 and msg in err, (rc, err)
    assert _lib.load().olb_irradiance_f32(None, None) == -1


def test_abi_accepts_an_empty_batch_without_device_work():
    assert _call(n_rays=0)[0] == 0


# ---- live reference: the plugin's wrapper against the reference's own body ---------------------------------------------

def _detector_system(be, extent=(-2.5, 2.5, -2.5, 2.5), **pose):
    from optiland.optic import Optic
    from optiland.physical_apertures import RectangularAperture

    op = Optic()
    op.surfaces.add(index=0, thickness=be.inf)
    op.surfaces.add(index=1, thickness=0, is_stop=True)
    op.surfaces.add(index=2, thickness=10)
    op.surfaces.add(index=3, **pose)
    op.surfaces[-1].aperture = RectangularAperture(x_min=extent[0], x_max=extent[1], y_min=extent[2], y_max=extent[3])
    op.wavelengths.add(0.55)
    op.fields.set_type("angle")
    op.fields.add(y=0)
    op.set_aperture("EPD", 5.0)
    return op


@pytest.fixture(params=["devmath", pytest.param("cuda", marks=pytest.mark.gpu)])
def live(request):
    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be

    from optiland_b200 import plugin as P

    if request.param == "cuda":
        eng = P.CudaEngine()
    else:
        from oracle.irradiance_engines import IrradianceDeviceMathEngine

        eng = IrradianceDeviceMathEngine()
    be.set_backend("torch")
    be.set_precision("float64")
    be.grad_mode.disable()
    if request.param == "cuda":
        be.set_device("cuda")
    yield P, eng, be, request.param
    if P._state.get("installed"):
        P.uninstall()
    be.set_backend("torch")
    be.set_precision("float64")
    be.grad_mode.disable()
    be.set_device("cpu")
    be.set_backend("numpy")


def _run(P, eng, make, install):
    """(data, stdout, (npix_x, npix_y)) of ``make()`` with the plugin installed over ``eng`` or not installed."""
    if install:
        P.install(engine=eng)
        P.stats(reset=True)
    elif P._state.get("installed"):
        P.uninstall()
    out = io.StringIO()
    with redirect_stdout(out):
        a = make()
    return a, out.getvalue()


def _set_records(be, surf, x, y, z, p):
    surf.x, surf.y, surf.z, surf.intensity = (be.array(v) for v in (x, y, z, p))


def _np(be, t):
    return np.asarray(be.to_numpy(t), dtype=np.float64)


def _compare(be, got, want, exact=True, slack=0.0):
    (g, gx, gy), (w, wx, wy) = got, want
    assert np.array_equal(gx, wx) and np.array_equal(gy, wy)
    assert type(g) is type(w) and g.dtype == w.dtype and g.device == w.device and g.requires_grad == w.requires_grad
    g, w = _np(be, g), _np(be, w)
    assert g.shape == w.shape
    if exact:
        np.testing.assert_allclose(g, w, rtol=1e-12, atol=1e-12 * max(1.0, float(np.abs(w).max())))
    else:
        assert float(np.abs(g - w).sum()) <= 2 * slack + 1e-12 * float(np.abs(w).sum()), (np.abs(g - w).sum(), slack)


@needs_ref
@pytest.mark.parametrize("precision", ["float64", "float32"])
@pytest.mark.parametrize("px_size", [None, (0.3, 0.7)])
@pytest.mark.parametrize("pose", [{}, {"dx": 0.31, "dy": -0.17}])
def test_skip_trace_wrapper_equals_reference(live, precision, px_size, pose):
    """IncoherentIrradiance(skip_trace=True) on adversarial detector records: the same map, edges, dtype, device, printed
    warning and npix update as the reference's body, one irradiance call on the engine, no decline."""
    from optiland.analysis import IncoherentIrradiance

    P, eng, be, which = live
    be.set_precision(precision)
    op = _detector_system(be, **pose)
    surf = op.surfaces[-1]
    dt = np.float64 if precision == "float64" else np.float32
    x0, y0 = float(pose.get("dx", 0.0)), float(pose.get("dy", 0.0))
    xe, ye = np.linspace(-2.5, 2.5, 11), np.linspace(-2.5, 2.5, 11)
    x, y, p = _samples(xe + x0, ye + y0, dt)
    _set_records(be, surf, x, y, np.zeros_like(x), p)

    def make():
        a = IncoherentIrradiance(op, res=(10, 10), px_size=px_size, skip_trace=True)
        return a.data[0][0], (a.npix_x, a.npix_y)

    (got, npix_g), out_g = _run(P, eng, make, True)
    assert not P.stats(), P.stats()
    assert eng.calls and eng.calls[-1][0] == "irradiance"
    (want, npix_w), out_w = _run(P, eng, make, False)
    assert out_g == out_w and npix_g == npix_w
    _compare(be, got, want)


@needs_ref
@pytest.mark.parametrize("precision", ["float64", "float32"])
def test_tilted_detector_within_edge_tolerance(live, precision):
    """A tilted, decentred detector: the kernel localizes with the effective (t, R) in fp64; a ray may change pixel only
    when its reference local coordinate lies within 1e-12 x scale (fp64) or 4 fp32 ulps of an edge."""
    from optiland.analysis import IncoherentIrradiance
    from optiland.visualization.system.utils import transform

    P, eng, be, which = live
    be.set_precision(precision)
    op = _detector_system(be, dx=0.2, dy=-0.1, rx=0.05, ry=-0.08)
    surf = op.surfaces[-1]
    dt = np.float64 if precision == "float64" else np.float32
    rng = np.random.default_rng(7)
    n = 20000
    x, y = rng.uniform(-3, 3, n).astype(dt), rng.uniform(-3, 3, n).astype(dt)
    z = rng.uniform(-0.3, 0.3, n).astype(dt)
    p = rng.uniform(0.1, 1.0, n).astype(dt)
    _set_records(be, surf, x, y, z, p)

    def make():
        return IncoherentIrradiance(op, res=(16, 12), skip_trace=True).data[0][0]

    got, _ = _run(P, eng, make, True)
    assert not P.stats(), P.stats()
    want, _ = _run(P, eng, make, False)
    xl, yl, _ = transform(surf.x, surf.y, surf.z, surf, is_global=True)
    xl, yl = _np(be, xl), _np(be, yl)
    near = np.zeros(n, dtype=bool)
    for v, e in ((xl, want[1]), (yl, want[2])):
        d = np.min(np.abs(v[:, None] - e[None, :]), axis=1)
        tol = 1e-12 * 3.0 if dt == np.float64 else 4 * np.spacing(np.abs(v).astype(np.float32)).astype(np.float64)
        near |= d <= tol
    slack = float(p[near].astype(np.float64).sum()) / float(want[1][1] - want[1][0]) / float(want[2][1] - want[2][0])
    _compare(be, got, want, exact=False, slack=slack)


@needs_ref
def test_fallbacks_record_a_reason(live):
    """Grad mode, an engine without ``irradiance`` and a degenerate extent hand the call to the reference's body, each
    with a reason; the reference's own result (or error) follows."""
    from optiland.analysis import IncoherentIrradiance

    from oracle.devmath_engine import DeviceMathEngine

    P, eng, be, which = live
    if which == "cuda":
        pytest.skip("host-side decisions; covered on the CPU")
    op = _detector_system(be)
    surf = op.surfaces[-1]
    x, y, p = _samples(*_edges("linspace"), np.float64)
    _set_records(be, surf, x, y, np.zeros_like(x), p)

    def make():
        return IncoherentIrradiance(op, res=(6, 6), skip_trace=True).data[0][0]

    def outcome(install, engine):
        try:
            r, _ = _run(P, engine, make, install)
            return ("ok", _np(be, r[0]))
        except Exception as e:   # the reference's error, whatever it is
            return ("error", type(e).__name__)

    be.grad_mode.enable()
    try:
        got = outcome(True, eng)
        assert P.stats() == {"irradiance: gradients wanted (bilinear branch)": 1}
        want = outcome(False, eng)
    finally:
        be.grad_mode.disable()
    assert got[0] == want[0] and np.array_equal(got[1], want[1], equal_nan=True)

    got = outcome(True, DeviceMathEngine())
    assert P.stats() == {"irradiance: engine has no irradiance kernel": 1}
    want = outcome(False, eng)
    assert got[0] == "ok" and np.array_equal(got[1], want[1], equal_nan=True)

    op.surfaces[-1].aperture.x_max = op.surfaces[-1].aperture.x_min = 0.5
    got = outcome(True, eng)
    assert P.stats() == {"irradiance: degenerate detector edges": 1}
    want = outcome(False, eng)
    assert got[0] == want[0]
    if got[0] == "ok":
        assert np.array_equal(got[1], want[1], equal_nan=True)
    else:
        assert got[1] == want[1]


@needs_ref
@pytest.mark.parametrize("power_dtype", ["float64", "list"])
def test_declined_rays_binned_the_reference_way(live, power_dtype):
    """Rays the engine does not take -- fp64 power with fp32 positions (narrowing it would change the weights), or a
    power that is not a tensor -- are binned by the wrapper's host path without tracing again: the reference's map,
    dtype and device, with a reason."""
    import torch
    from optiland.analysis import IncoherentIrradiance

    P, eng, be, which = live
    be.set_precision("float32")
    op = _detector_system(be, dx=0.31, dy=-0.17)
    surf = op.surfaces[-1]
    x, y, p = _samples(np.linspace(-2.2, 2.8, 11), np.linspace(-2.7, 2.3, 11), np.float32)
    _set_records(be, surf, x, y, np.zeros_like(x), p)
    p64 = np.random.default_rng(5).uniform(-0.5, 2.0, x.size)
    dev = surf.x.device
    surf.intensity = torch.tensor(p64, dtype=torch.float64, device=dev) if power_dtype == "float64" else p64.tolist()

    def make():
        return IncoherentIrradiance(op, res=(10, 10), skip_trace=True).data[0][0]

    if power_dtype == "list":
        # a list power breaks the reference's own body (be.to_numpy / the mask); the wrapper must raise the same way
        def outcome(install):
            try:
                _run(P, eng, make, install)
                return "ok"
            except Exception as e:
                return type(e).__name__
        got = outcome(True)
        assert P.stats() == {"irradiance: rays not accepted by the engine": 1}
        assert got == outcome(False)
        return
    got, _ = _run(P, eng, make, True)
    assert P.stats() == {"irradiance: rays not accepted by the engine": 1}
    assert not any(c[0] == "irradiance" for c in eng.calls if c)
    want, _ = _run(P, eng, make, False)
    _compare(be, got, want)


# ---- GPU: the kernel itself ----------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["float64", "float32"])
@pytest.mark.parametrize("kind", ["linspace", "arange"])
@pytest.mark.parametrize("path", ["shared", "global", "auto_large"])
def test_kernel_matches_histogram2d(dtype, kind, path):
    """Adversarial samples through olb_irradiance_*: identical bins to np.histogram2d (each sample alone), sums to
    1e-12, on each accumulation path (forced on the small grid; a grid over 27 x 1024 bins takes the global one)."""
    import torch

    from optiland_b200.irradiance import bin_irradiance

    dt = np.float64 if dtype == "float64" else np.float32
    force = {"shared": _lib.IRR_PATH_SHARED, "global": _lib.IRR_PATH_GLOBAL, "auto_large": _lib.IRR_PATH_AUTO}[path]
    if path != "auto_large":
        xe, ye = _edges(kind)
    else:
        xe, ye = np.linspace(-2.5, 2.5, 301), np.linspace(-1.0, 3.0, 201)
    x, y, p = _samples(xe, ye, dt)
    tx, ty, tp = (torch.from_numpy(v).cuda() for v in (x, y, p))
    hist = bin_irradiance(tx, ty, tp, xe, ye, path=force).cpu().numpy()
    np.testing.assert_allclose(hist, _histogram2d(x, y, p, xe, ye), rtol=1e-12, atol=0)
    # bin indices: every ray alone, read back from the one non-zero cell
    want = _reference_bins(x, y, p, xe, ye)
    sel = np.concatenate([np.flatnonzero(want >= 0)[:300], np.flatnonzero(want < 0)[:60]])
    ones = torch.ones(1, dtype=tx.dtype, device="cuda")
    for r in sel:
        h = bin_irradiance(tx[r:r + 1], ty[r:r + 1], tp[r:r + 1].clone() if p[r] <= 0 or np.isnan(p[r]) else ones, xe, ye,
                           path=force)
        nz = torch.nonzero(h.reshape(-1)).reshape(-1).cpu().numpy()
        assert (nz.tolist() or [-1]) == [want[r]], (r, x[r], y[r], p[r])


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["float64", "float32"])
@pytest.mark.parametrize("path", ["auto", "shared", "global"])
def test_kernel_focused_beam(dtype, path):
    """10^6 rays into the four pixels around one vertex of a 21 x 21 grid (the contention case the warp grouping is
    for): exact counts on either path, with and without rays that are dropped in the same warps."""
    import torch

    from optiland_b200.irradiance import bin_irradiance

    force = {"auto": _lib.IRR_PATH_AUTO, "shared": _lib.IRR_PATH_SHARED, "global": _lib.IRR_PATH_GLOBAL}[path]
    dt = torch.float64 if dtype == "float64" else torch.float32
    n = 1_000_000
    xe = ye = np.linspace(-2.5, 2.5, 22)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = float(xe[11]) + (torch.rand(n, device="cuda", generator=g, dtype=dt) - 0.5) * 0.2
    y = float(ye[11]) + (torch.rand(n, device="cuda", generator=g, dtype=dt) - 0.5) * 0.2
    p = torch.ones(n, device="cuda", dtype=dt)
    p[5::9] = 0                     # dropped lanes share warps with the colliding ones
    hist = bin_irradiance(x, y, p, xe, ye, path=force).cpu().numpy()
    want = _histogram2d(x.cpu().numpy(), y.cpu().numpy(), p.cpu().numpy(), xe, ye)
    assert np.count_nonzero(want) == 4
    assert np.array_equal(hist, want) and hist.sum() == float(p.sum())


# ---- GPU: the live analysis end to end -----------------------------------------------------------------------------------

@needs_ref
@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["float64", "float32"])
@pytest.mark.parametrize("how", ["trace", "user_rays", "source"])
def test_incoherent_irradiance_on_cuda_equals_reference(precision, how):
    """The unmodified IncoherentIrradiance on a CUDA torch backend: plugin against stock.  The trace path, user rays and
    an SMFSource; the kernel really ran (launch count) and nothing declined."""
    import torch

    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be
    from optiland.analysis import IncoherentIrradiance
    from optiland.rays import RealRays

    from optiland_b200 import plugin as P

    be.set_backend("torch")
    be.set_device("cuda")
    be.set_precision(precision)
    be.grad_mode.disable()
    try:
        op = _detector_system(be)

        def make():
            torch.manual_seed(0)
            if how == "trace":
                a = IncoherentIrradiance(op, num_rays=200_000, res=(64, 64), distribution="random")
            elif how == "user_rays":
                n = 300_000
                g = torch.Generator(device="cuda").manual_seed(1)
                dt = torch.float64 if precision == "float64" else torch.float32
                x = (torch.rand(n, generator=g, device="cuda", dtype=dt) - 0.5) * 6
                y = (torch.rand(n, generator=g, device="cuda", dtype=dt) - 0.5) * 6
                z0 = torch.zeros(n, device="cuda", dtype=dt)
                rays = RealRays(x, y, z0, z0, z0, z0 + 1, torch.rand(n, generator=g, device="cuda", dtype=dt),
                                z0 + 0.55)
                a = IncoherentIrradiance(op, res=(50, 40), user_initial_rays=rays)
            else:
                from optiland.sources import SMFSource

                src = SMFSource(mfd_um=10.4, wavelength_um=0.55, position=(0.0, 0.0, -5.0))
                a = IncoherentIrradiance(op, num_rays=100_000, res=(32, 32), source=src)
            return a.data[0][0]

        from optiland_b200 import _lib

        eng = P.CudaEngine()
        l0 = _lib.load().olb_launch_count()
        got, _ = _run(P, eng, make, True)
        why = P.stats()
        n_irr = sum(1 for c in eng.calls if c[0] == "irradiance")
        want, _ = _run(P, eng, make, False)
        if how == "source" and n_irr == 0:
            # the source's rays are not device-resident: the wrapper bins them the reference's way (compared below)
            assert "irradiance: rays not accepted by the engine" in why, why
        else:
            assert not why, why
            assert n_irr == 1 and _lib.load().olb_launch_count() > l0
        # same traced rays on both sides (the plugin's trace equals the reference's to rounding): the maps may differ
        # only by rays within rounding of an edge
        g, w = _np(be, got[0]), _np(be, want[0])
        assert g.shape == w.shape and np.array_equal(got[1], want[1])
        assert got[0].dtype == want[0].dtype and got[0].device == want[0].device
        assert float(np.abs(g - w).sum()) <= 1e-6 * float(np.abs(w).sum()) + 1e-9, float(np.abs(g - w).sum())
    finally:
        if P._state.get("installed"):
            P.uninstall()
        be.set_precision("float64")
        be.set_device("cpu")
        be.set_backend("numpy")


@needs_ref
@pytest.mark.gpu
@pytest.mark.timeout(1500)
def test_reference_irradiance_tests_on_cuda_grad_mode_off():
    """The reference's own IncoherentIrradiance tests (torch backend on the GPU, grad mode off), stock against the plugin
    over the product engine: the same passing set, and the irradiance kernel carried calls."""
    from oracle.ref_import import REFERENCE_ROOT, REFERENCE_TESTS

    def run(install):
        env = dict(os.environ, OLB_SWEEP_INSTALL="1" if install else "0", PYTHONPATH=ROOT, OLB_SWEEP_NOGRAD="1",
                   OLB_SWEEP_DEVICE="cuda")
        with tempfile.TemporaryDirectory(prefix="olb_irr_") as rootdir:
            out = subprocess.run(
                [sys.executable, "-m", "pytest", "-p", "oracle.sweep_plugin", "-p", "oracle.sweep_irradiance", "-p",
                 "no:cacheprovider", "-q", "--no-header", "-rfE", f"--rootdir={rootdir}",
                 f"--confcutdir={REFERENCE_ROOT}", "-c", "/dev/null", os.path.join(REFERENCE_TESTS, "test_analysis.py"),
                 "-k", "IncoherentIrradiance and torch"],
                cwd=rootdir, env=env, capture_output=True, text=True, timeout=1400).stdout
        bad = set(re.findall(r"^(?:FAILED|ERROR) (\S+)", out, flags=re.M))
        counts = {k: int(v) for v, k in re.findall(r"(\d+) (passed|failed|error)", out)}
        m = re.search(r"\[olb sweep\] irradiance calls: (\d+)", out)
        return counts, bad, int(m.group(1)) if m else 0, out

    stock, bad_stock, _, _ = run(False)
    ours, bad_ours, n_irr, log = run(True)
    print(f"stock {stock} | plugin {ours} | irradiance calls {n_irr}")
    assert stock.get("passed", 0) > 0
    assert bad_ours == bad_stock and ours == stock, (stock, ours, sorted(bad_ours ^ bad_stock))
    assert n_irr > 0, log[-3000:]
