"""Forbes Q-2D freeform surfaces (Optiland's ``surface_type="forbes_q2d"``, ``ForbesQ2dGeometry``) on the trace path: the
C ABI and table layer, the kernel arithmetic against fixtures the unmodified reference produced (tests/golden/forbes_q2d,
``oracle/make_golden_forbes_q2d.py``), the plugin with live reference objects, and what stays declined.  GPU tests are
marked; the rest runs on the CPU through the host instantiation of the device arithmetic with the Q-2D kernel variants
(tests/hostcheck/hostcheck_forbes_q2d.cpp), its NumPy restatement (oracle/forbes_q2d_oracle.py) and the test engines
built on them (oracle/forbes_q2d_engines.py)."""
import ctypes as C
import glob
import json
import os

import numpy as np
import pytest

from optiland_b200 import table as T
from tests._util import GOLDEN, REC, Case, fp32_errors, max_abs_err

Q2D_CASES = sorted("forbes_q2d/" + os.path.splitext(os.path.basename(p))[0]
                   for p in glob.glob(os.path.join(GOLDEN, "forbes_q2d", "*.npz")))
PLAIN_CASES = [c for c in Q2D_CASES if "polarized" not in c]
FEAT_Q2D = 1 << 11


def _bounds(name):
    with open(os.path.join(GOLDEN, "forbes_q2d", "f32_achieved.json")) as f:
        return json.load(f)["cases"][name.split("/", 1)[1]]


def _pmat(c, dtype=np.complex128):
    return np.tile(np.eye(3, dtype=dtype), (c.n, 1, 1)) if "out_p" in c.z else None


def _q2d(cm0=(1e-3, -2e-3), ams=((2e-3, 1e-3, 0, 5e-4), (1e-3,)), bms=((-1e-3,), ()), **kw):
    kw.setdefault("t", [0, 0, 1.0])
    return T.SurfaceSpec(kind=T.GEOM_FORBES_Q2D, n1=[1.0], n2=[1.5], radius=kw.pop("radius", -40.0),
                         norm_radius=kw.pop("norm_radius", 5.0), q2d_cm0=cm0, q2d_ams=list(ams), q2d_bms=list(bms),
                         tol=1e-12, **kw)


def _table(*specs):
    return T.SurfaceTable([T.SurfaceSpec(kind=T.GEOM_NOOP)] + list(specs), [0.55])


def _raw_upload_codes(tab, mutate):
    """olb_table_workspace_bytes / the host check's feature word on a table whose packed arrays ``mutate`` edits."""
    from optiland_b200 import _lib
    from oracle.hostcheck_api import load

    surf, pool = tab.pack()
    mutate(surf, pool)
    ht = _lib.HostTable(tab, packed=(surf, pool))
    lib = _lib.load()
    rc = int(lib.olb_table_workspace_bytes(C.byref(ht.c)))
    buf = C.create_string_buffer(256)
    lib.olb_last_error(buf, 256)
    return rc, buf.value.decode(), int(load().olbhc_features(C.byref(ht.c)))


# ---- ABI / table layer -----------------------------------------------------------------------------------------

def test_abi_constants_and_version_unchanged():
    from optiland_b200 import _lib

    assert T.GEOM_FORBES_Q2D == 12 and T.OLB_SURFACE_DTYPE.itemsize == 192
    assert (T.Q2D_MAX_M, T.Q2D_MAX_TERMS, T.MAX_Q2D_ELEMENTS) == (16, 16, 4096)
    assert _lib.load().olb_version() == 3
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "olb.h")).read()
    for name, v in (("OLB_GEOM_FORBES_Q2D", 12), ("OLB_Q2D_MAX_M", 16), ("OLB_Q2D_MAX_TERMS", 16), ("OLB_MAX_Q2D_ELEMENTS", 4096)):
        assert f"#define {name}" in hdr and str(v) in hdr.split(f"#define {name}")[1].split("\n")[0]


def test_q2d_block_layout_and_round_trip():
    """pack writes cm0, {na_m, nb_m} x M and the lists a_1, b_1, a_2, b_2 at coef_off with aux0 = n0 and n_coef = M;
    unpack gives the table back (what the distributed table broadcast sends)."""
    tab = _table(_q2d(max_iter=7), T.SurfaceSpec(kind=T.GEOM_STANDARD, radius=-40.0, t=[0, 0, 5.0]))
    surf, pool = tab.pack()
    assert (surf["kind"][1], surf["aux0"][1], surf["n_coef"][1], surf["max_iter"][1]) == (T.GEOM_FORBES_Q2D, 2, 2, 7)
    assert surf["norm_radius"][1] == 5.0 and surf["radius"][1] == -40.0
    o = surf["coef_off"][1]
    want = [1e-3, -2e-3, 4, 1, 1, 0, 2e-3, 1e-3, 0, 5e-4, -1e-3, 1e-3]
    assert list(pool[o:o + len(want)]) == want
    back = T.SurfaceTable.unpack(surf, pool, tab.wavelengths)
    g = back.surfaces[1]
    assert np.array_equal(g.q2d_cm0, [1e-3, -2e-3]) and len(g.q2d_ams) == 2 and len(g.q2d_bms) == 2
    assert np.array_equal(g.q2d_ams[0], [2e-3, 1e-3, 0, 5e-4]) and np.array_equal(g.q2d_bms[1], [])
    assert back.content_key() == tab.content_key()
    for bad, word in ((dict(cm0=[np.nan]), "non-finite"), (dict(ams=[[0.0] * 17], bms=[[]]), "longer"),
                      (dict(ams=[[]] * 17, bms=[[]] * 17), "at most"), (dict(ams=[[1.0]], bms=[]), "sine"),
                      (dict(norm_radius=0.0), "norm_radius")):
        with pytest.raises(ValueError, match=word):
            _table(_q2d(**bad))


def test_q2d_element_cap():
    """The Q-2D blocks of one table are staged in shared memory: at most MAX_Q2D_ELEMENTS prepared elements; three
    surfaces at the caps fit, a fourth does not -- in the table layer and in the upload's own check."""
    full = dict(cm0=[1e-4] * 16, ams=[[1e-4] * 16] * 16, bms=[[1e-4] * 16] * 16)
    assert T.q2d_elements(full["cm0"], full["ams"], full["bms"]) == 1364
    three = [_q2d(**full, t=[0, 0, z]) for z in (1.0, 2.0, 3.0)]
    ok = _table(*three)
    with pytest.raises(ValueError, match="shared memory"):
        _table(*three, _q2d(**full, t=[0, 0, 4.0]))
    assert _raw_upload_codes(ok, lambda s, p: None)[0] > 0
    four = object.__new__(T.SurfaceTable)          # (past the table layer's own check)
    four.surfaces = ok.surfaces + [_q2d(**full, t=[0, 0, 4.0])]
    four.wavelengths = ok.wavelengths
    rc, msg, _ = _raw_upload_codes(four, lambda s, p: None)
    assert rc == -5 and "4096" in msg and "shared memory" in msg


def test_malformed_q2d_blocks_are_table_errors():
    tab = _table(_q2d())
    rc, msg, feat = _raw_upload_codes(tab, lambda s, p: None)
    assert rc > 0 and feat & FEAT_Q2D

    def off(s):
        return int(s["coef_off"][1])

    def big_m(s, p):
        s["n_coef"][1] = 17

    def big_n0(s, p):
        s["aux0"][1] = 17

    def frac_len(s, p):
        p[off(s) + 2] = 1.5

    def long_list(s, p):
        p[off(s) + 2] = 17

    def nan_coef(s, p):
        p[off(s) + 6] = np.nan

    def zero_norm(s, p):
        s["norm_radius"][1] = 0.0

    def outside(s, p):
        s["coef_off"][1] = len(p) - 4

    def negative_iter(s, p):
        s["max_iter"][1] = -1

    for mutate, word in ((big_m, "M out of range"), (big_n0, "bad Forbes Q-2D block"), (frac_len, "integers"),
                         (long_list, "integers"), (nan_coef, "non-finite"), (zero_norm, "norm_radius"),
                         (outside, "Forbes Q-2D block"), (negative_iter, "max_iter")):
        rc, msg, feat = _raw_upload_codes(tab, mutate)
        assert rc == -5 and word in msg and feat == -1, (mutate.__name__, rc, msg)


def test_no_adjoint_and_batched_uploads_refuse_q2d_tables():
    from optiland_b200 import _lib
    from optiland_b200.batch import template_params
    from oracle.hostcheck_api import load

    tab = _table(_q2d())
    ht = _lib.HostTable(tab)
    hc = load()
    assert hc.olbhc_bwd_supported(C.byref(ht.c)) == 0
    params = np.zeros((2, tab.num_surfaces, _lib.BP_COUNT))
    err = C.create_string_buffer(256)
    out = np.zeros(1 << 16, dtype=np.uint8)
    feat = C.c_uint(0)
    rc = hc.olbhc_batch_blob(C.byref(ht.c), C.c_void_p(params.ctypes.data), 2, 0, 0, C.c_void_p(out.ctypes.data),
                             out.size, C.byref(feat), err, 256)
    assert rc == -1 and b"Q-2D" in err.value
    lib = _lib.load()
    ws = np.zeros(1 << 16, dtype=np.uint8)
    dt = _lib.OlbDeviceTable()
    rc = lib.olb_table_upload_batch(C.byref(ht.c), C.c_void_p(params.ctypes.data), 2,
                                    C.c_void_p((ws.ctypes.data + 15) & ~15), C.c_int64(ws.size - 16), None, C.byref(dt))
    assert rc == -2
    with pytest.raises(ValueError, match="Q-2D"):
        template_params(tab)


# ---- kernel arithmetic (host instantiation) vs the reference's fixtures ----------------------------------------

def _check_fp64(c, rec, out=None):
    tol = 1e-11 * c.scale
    for k in REC:
        assert max_abs_err(rec[k], c.rec[k]) <= tol, k      # (max_abs_err also asserts the same NaN pattern)
    assert np.array_equal(rec["intensity"] == 0, c.rec["intensity"] == 0)
    if out is not None and "p" in out:
        assert np.array_equal(np.isnan(out["p"]), np.isnan(c.out["p"]))
        assert np.nanmax(np.abs(out["p"] - c.out["p"])) <= 1e-11


@pytest.mark.parametrize("name", Q2D_CASES)
def test_host_arithmetic_fp64_matches_reference_fixture(name):
    from oracle.hostcheck_forbes_q2d import run_hostcheck_forbes_q2d

    c = Case(name)
    out, rec, status = run_hostcheck_forbes_q2d(c.table, c.rays, np.float64, pmat=_pmat(c), want_l0=True)
    assert status == 0
    _check_fp64(c, rec, out)
    for k in ("x", "y", "z", "L", "M", "N", "i", "opd", "L0", "M0", "N0"):
        assert max_abs_err(out[k], c.out[k]) <= 1e-11 * c.scale, k


@pytest.mark.parametrize("name", Q2D_CASES)
def test_host_arithmetic_fp32_as_measured(name):
    """The fp32 instantiation's error per fixture stays within 3x tests/golden/forbes_q2d/f32_achieved.json (the larger
    of this and the H100 kernel, scripts/f32_achieved_forbes_q2d.py)."""
    from oracle.hostcheck_forbes_q2d import run_hostcheck_forbes_q2d

    c = Case(name)
    out, rec, _ = run_hostcheck_forbes_q2d(c.table, c.rays, np.float32, pmat=_pmat(c, np.complex64))
    bound = _bounds(name)
    for k, v in fp32_errors(rec, c.rec).items():
        assert v <= 3.0 * bound[k] + 1e-12, (k, v, bound[k])


@pytest.mark.parametrize("name", Q2D_CASES)
def test_numpy_restatement_matches_reference_fixture(name):
    """oracle/forbes_q2d_oracle.py, the independent NumPy restatement the live tests use, reproduces every fixture."""
    from oracle import forbes_q2d_oracle as Q

    c = Case(name)
    pm = _pmat(c)
    inp = dict(c.rays, p=pm) if pm is not None else c.rays
    _, rec, _ = Q.trace(c.table, inp, polarized=pm is not None)
    _check_fp64(c, rec)


def test_m0_only_surface_equals_its_qbfs_twin():
    """A Q-2D surface with m = 0 terms only traces as the Q-bfs surface of the same terms, within the fp64 bound (not
    bit for bit: the Q-2D sag adds 1e-12 to r^2 before forming u)."""
    from oracle.hostcheck_forbes_q2d import run_hostcheck_forbes_q2d

    q2d, twin = Case("forbes_q2d/q2d_m0_only"), Case("forbes_q2d/q2d_m0_qbfs_twin")
    assert q2d.table.surfaces[2].kind == T.GEOM_FORBES_Q2D and twin.table.surfaces[2].kind == T.GEOM_FORBES_QBFS
    assert np.array_equal(q2d.rays["x"], twin.rays["x"])
    _, rec, _ = run_hostcheck_forbes_q2d(q2d.table, q2d.rays, np.float64)
    for k in REC:
        assert max_abs_err(rec[k], twin.rec[k]) <= 1e-11 * twin.scale, k


def test_fixtures_pin_the_reference_behaviours():
    """Vertex rays, rays on the axes and beyond u = 1, rays that miss (NaN from the base sphere on), and rays stopped by
    max_iter all appear in the fixtures the arithmetic is held to; the vertex rays leave with the reference's vertex
    slope, and the departure vanishes beyond the normalisation radius."""
    from oracle import forbes_q2d_oracle as Q

    v = Case("forbes_q2d/q2d_vertex")
    x, y = v.rays["x"], v.rays["y"]
    s = v.table.surfaces[1]
    on = (x == 0) & (y == 0)
    assert on.sum() >= 4 and np.all(np.isfinite(v.rec["x"][1]))
    vx, vy = Q.q2d_vertex_slopes(s)
    assert vx != 0 and vy != 0
    L, M = v.out["L0"], v.out["M0"]                  # (directions before the last surface's interaction)
    assert np.all(np.isfinite(L[on])) and len(np.unique(v.rec["L"][1][on])) == 1
    far = np.hypot(x, y) > 3.0 * (1 + 1e-10)
    assert far.sum() >= 48
    sag = v.rec["z"][1] - s.t[2]
    base = Q.q2d_sag(T.SurfaceSpec(kind=T.GEOM_FORBES_Q2D, radius=s.radius, conic=s.conic, norm_radius=s.norm_radius),
                     v.rec["x"][1][far], v.rec["y"][1][far])
    assert np.max(np.abs(sag[far] - base)) < 1e-12
    nan = Case("forbes_q2d/q2d_nan_rays")
    bad = np.isnan(nan.rec["x"][2])
    assert bad.any() and not bad.all() and np.all(np.isnan(nan.rec["x"][3][bad]))
    few, full = Case("forbes_q2d/q2d_max_iter"), Case("forbes_q2d/q2d_singlet")
    assert np.nanmax(np.abs(few.rec["z"][2] - full.rec["z"][2])) > 1e-9     # max_iter = 2 stops before convergence
    ho = Case("forbes_q2d/q2d_high_order").table.surfaces[2]
    assert len(ho.q2d_ams) == 8 and len(ho.q2d_ams[0]) == 6 and max(len(a) for a in ho.q2d_ams) == 10


def test_sag_and_slopes_against_the_reference_geometry():
    """The kernel's sag and slopes (host instantiation, fp64) against ForbesQ2dGeometry.sag / _surface_normal at random
    points, on the vertex (both signs of zero), on the normalisation circle and beyond it, for finite and infinite
    base radii."""
    pytest.importorskip("oracle.ref_import")
    from oracle.ref_import import import_reference, reference_available

    if not reference_available():
        pytest.skip("reference not present on this box")
    import_reference()
    import optiland.backend as be
    from optiland.coordinate_system import CoordinateSystem
    from optiland.geometries.forbes.geometry import ForbesQ2dGeometry, ForbesSolverConfig, ForbesSurfaceConfig

    from optiland_b200.pack import pack_forbes_q2d
    from oracle.hostcheck_forbes_q2d import eval_surface
    from tests._forbes_q2d_systems import freeform

    be.set_backend("numpy")
    rng = np.random.default_rng(4)
    x = np.concatenate([rng.uniform(-11, 11, 3000), [0.0, -0.0, 0.0, 1e-13, 0.0, 10.0, 0.0, -10.0]])
    y = np.concatenate([rng.uniform(-11, 11, 3000), [0.0, 0.0, -0.0, 0.0, 1e-13, 0.0, 10.0, 0.0]])
    for R, k in ((50.0, -0.5), (float("inf"), 0.0), (-80.0, 0.3)):
        g = ForbesQ2dGeometry(CoordinateSystem(), ForbesSurfaceConfig(radius=R, conic=k, norm_radius=10.0,
                                                                       terms=freeform(7, 8, 1e-3, 1, m1_terms=5)),
                              ForbesSolverConfig())
        spec = T.SurfaceSpec(kind=T.GEOM_FORBES_Q2D, radius=R, conic=k)
        pack_forbes_q2d(spec, g)
        spec.__post_init__()
        z, (nx, ny, nz) = g.sag(x, y), g._surface_normal(x, y)
        sag, fx, fy = eval_surface(_table(spec), 1, x, y)
        assert np.max(np.abs(sag - z)) <= 1e-14 * max(1.0, np.max(np.abs(z)))
        assert np.max(np.abs(fx - nx / -nz)) <= 1e-14 and np.max(np.abs(fy - ny / -nz)) <= 1e-14


# ---- engines: the plugin with live reference objects -----------------------------------------------------------

pytest_ref = pytest.importorskip("oracle.ref_import")
needs_ref = pytest.mark.skipif(not pytest_ref.reference_available(), reason="reference not present on this box")

LIVE_REC = ("x", "y", "z", "L", "M", "N", "opd", "intensity")


@pytest.fixture(params=["devmath", "oracle", pytest.param("cuda", marks=pytest.mark.gpu)])
def live(request):
    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be

    from optiland_b200 import plugin as P

    if request.param == "cuda":
        eng = P.CudaEngine()
    elif request.param == "oracle":
        from oracle.forbes_q2d_engines import Q2dOracleEngine

        eng = Q2dOracleEngine()
    else:
        from oracle.forbes_q2d_engines import Q2dDeviceMathEngine

        eng = Q2dDeviceMathEngine()
    yield P, eng, be, request.param
    if P._state.get("installed"):
        P.uninstall()
    be.set_backend("torch")
    be.grad_mode.disable()
    if request.param == "cuda":
        be.set_device("cpu")
    be.set_backend("numpy")


def _install(P, eng, be, which):
    be.set_backend("torch")
    be.set_precision("float64")
    be.grad_mode.disable()
    if which == "cuda":
        be.set_device("cuda")
    P.install(engine=eng)
    P.stats(reset=True)


def _close(got, want, scale, what):
    assert got.shape == want.shape, what
    assert np.array_equal(np.isnan(got), np.isnan(want)), (what, "NaN pattern")
    m = np.isfinite(want)
    assert not m.any() or np.max(np.abs(got[m] - want[m])) <= 1e-11 * scale, (what, float(np.max(np.abs(got[m] - want[m]))))


@needs_ref
@pytest.mark.parametrize("system", ["q2d_singlet", "q2d_high_order", "q2d_nested_reflection", "q2d_nan_rays",
                                    "q2d_aperture_coating", "q2d_polarized", "q2d_infinite_radius"])
def test_optic_trace_through_the_plugin_equals_the_reference(live, system):
    """Optic.trace of two fields x every wavelength: each record row equals the NumPy reference, in one fused launch
    per trace, no decline."""
    from tests import _forbes_q2d_systems as QS

    P, eng, be, which = live
    be.set_backend("numpy")
    ref = QS.BUILDERS[system](be)
    wls = [float(w.value) for w in ref.wavelengths.wavelengths]
    jobs = [(hy, wl) for hy in (0.0, 1.0) for wl in wls]
    want = []
    for hy, wl in jobs:
        r = ref.trace(0.0, hy, wl, 10, "hexapolar")
        want.append(({k: np.array(getattr(ref.surfaces, k)) for k in LIVE_REC}, np.array(r.i)))
    _install(P, eng, be, which)
    lens = QS.BUILDERS[system](be)
    n0 = len(eng.calls)
    for (hy, wl), (w, wi) in zip(jobs, want):
        r = lens.trace(0.0, hy, wl, 10, "hexapolar")
        scale = max(1.0, float(np.nanmax(np.abs(w["z"]))))
        for k, v in w.items():
            _close(be.to_numpy(getattr(lens.surfaces, k)), v, scale, k)
        _close(be.to_numpy(r.i), wi, 1.0, "i")
    assert not P.stats(), P.stats()
    assert sum(1 for c in eng.calls[n0:] if c and c[0] == "pupil") == len(jobs), eng.calls[n0:]


@needs_ref
def test_trace_generic_spot_diagram_and_wavefront(live):
    """trace_generic with per-ray fields and wavelengths, SpotDiagram.rms_spot_radius and the Wavefront OPD map of the
    gallery singlet equal the NumPy reference with no decline."""
    from optiland.analysis import SpotDiagram
    from optiland.wavefront import Wavefront

    from tests import _forbes_q2d_systems as QS

    P, eng, be, which = live
    rng = np.random.default_rng(11)
    n = 300
    Hx, Hy = rng.uniform(-0.3, 0.3, n), rng.uniform(0, 1, n)
    Px, Py = rng.uniform(-0.7, 0.7, n), rng.uniform(-0.7, 0.7, n)
    wl = rng.choice(list(QS.WL3), n)

    def run(lens):
        out = {}
        r = lens.trace_generic(be.array(Hx), be.array(Hy), be.array(Px), be.array(Py), be.array(wl))
        for k in ("x", "y", "z", "L", "M", "N", "i", "opd"):
            out["g_" + k] = np.array(be.to_numpy(getattr(r, k)), dtype=np.float64)
        out["rms"] = np.array([[float(be.to_numpy(v)) for v in row] for row in SpotDiagram(lens).rms_spot_radius()])
        wf = Wavefront(lens, fields=[(0.0, 0.0), (0.0, 0.7)], wavelengths=[0.5876], num_rays=8, distribution="hexapolar")
        for j, d in enumerate(wf.data.values()):
            out[f"wf{j}_opd"] = np.array(be.to_numpy(d.opd), dtype=np.float64)
            out[f"wf{j}_i"] = np.array(be.to_numpy(d.intensity), dtype=np.float64)
        return out

    be.set_backend("numpy")
    want = run(QS.singlet(be))
    _install(P, eng, be, which)
    got = run(QS.singlet(be))
    for k, v in want.items():
        np.testing.assert_allclose(got[k], v, rtol=1e-9 if k == "rms" else 0, atol=0 if k == "rms" else 1e-9, err_msg=k)
    assert not P.stats(), P.stats()


@needs_ref
def test_declined_q2d_configurations():
    """A subclass of ForbesQ2dGeometry, lists over the caps, non-finite coefficients and a Q-2D surface beside a phase
    profile, a grid sag, a BSDF or a thin-film coating each decline with a reason."""
    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be

    from optiland_b200.pack import UnsupportedSurface, pack_surface_group
    from tests import _forbes_q2d_systems as QS

    be.set_backend("numpy")
    tab = pack_surface_group(QS.singlet(be).surfaces, [0.55])
    s = tab.surfaces[2]
    assert s.kind == T.GEOM_FORBES_Q2D and s.norm_radius == 10.0 and len(s.q2d_ams) == 1
    assert np.array_equal(s.q2d_cm0, [1.0, 0, 0, 0, 4.0]) and list(s.q2d_ams[0]) == [0.0, 2.0]
    lens = QS.singlet(be)
    g = lens.surfaces.surfaces[2].geometry
    g.__class__ = type("MyQ2d", (type(g),), {})
    with pytest.raises(UnsupportedSurface, match="MyQ2d"):
        pack_surface_group(lens.surfaces, [0.55])

    def edited(changes):
        lens = QS.singlet(be)
        g = lens.surfaces.surfaces[2].geometry
        g.freeform_coeffs.update(changes)
        g._prepare_coeffs()
        return lens

    with pytest.raises(UnsupportedSurface, match="radial order"):
        pack_surface_group(edited({("a", 0, 16): 1e-6}).surfaces, [0.55])
    with pytest.raises(UnsupportedSurface, match="azimuthal order"):
        pack_surface_group(edited({("b", 17, 0): 1e-6}).surfaces, [0.55])
    with pytest.raises(UnsupportedSurface, match="non-finite"):
        pack_surface_group(edited({("a", 2, 1): float("nan")}).surfaces, [0.55])
    from optiland.phase import RadialPhaseProfile

    lens = QS.singlet(be)
    lens.surfaces.add(index=3, radius=be.inf, thickness=5.0, phase_profile=RadialPhaseProfile([-1.0]))
    with pytest.raises(UnsupportedSurface, match="beside a phase profile"):
        pack_surface_group(lens.surfaces, [0.55])
    from optiland.scatter import LambertianBSDF

    lens = QS.singlet(be)
    lens.surfaces.surfaces[1].interaction_model.bsdf = LambertianBSDF()
    with pytest.raises(UnsupportedSurface, match="beside a BSDF"):
        pack_surface_group(lens.surfaces, [0.55])


@needs_ref
def test_gradients_and_coefficient_variables_decline_to_the_reference(live):
    """With grad mode on, or a ForbesQ2dCoeffVariable driving a coefficient, the trace declines with a reason in
    plugin.stats() and returns the reference's results and gradients."""
    import torch
    from optiland.optimization.variable.forbes_coeff import ForbesQ2dCoeffVariable

    from tests import _forbes_q2d_systems as QS

    P, eng, be, which = live
    if which == "oracle":
        pytest.skip("one engine suffices: the reference's eager path runs")

    def run():
        be.grad_mode.enable()
        lens = QS.m0_only(be)
        var = ForbesQ2dCoeffVariable(lens, 2, ("a", 1, 1))
        v = torch.tensor(1e-3, dtype=torch.float64, requires_grad=True)
        var.update_value(v * 1.0)
        lens.trace(0.0, 0.7, 0.5876, 6, "hexapolar")
        y = lens.surfaces.y[-1]
        loss = torch.nansum(y * y)
        loss.backward()
        be.grad_mode.disable()
        return float(loss.detach()), float(v.grad)

    be.set_backend("torch")
    be.set_precision("float64")
    if which == "cuda":
        be.set_device("cuda")
    want = run()
    _install(P, eng, be, which)
    got = run()
    assert np.isfinite(want[1]) and want[1] != 0
    assert got[0] == pytest.approx(want[0], rel=1e-12) and got[1] == pytest.approx(want[1], rel=1e-9)
    assert P.stats(), "the gradient trace must decline"
    assert not any(c and c[0] == "pupil" for c in eng.calls)


@needs_ref
def test_device_aiming_declines_on_q2d_tables(live):
    """Robust ray aiming never launches the aim kernel on a table with a Q-2D surface before the stop: the solver
    declines with a reason, the reference's aimer runs (with the plugin's fused subset traces) and gives the reference's
    rays."""
    from tests import _forbes_q2d_systems as QS

    P, eng, be, which = live
    if which == "oracle":
        pytest.skip("one engine suffices")
    if not hasattr(eng, "aim"):
        def aim(*a, **k):
            raise AssertionError("the aim kernel must not run on a Q-2D table")

        eng.aim = aim

    def build(be):
        lens, done = QS._lens(be, 10.0, (0.0, 10.0), (0.5876,))
        lens.surfaces.add(index=1, radius=be.inf, thickness=3.0, material="N-BK7", tol=1e-12,
                          **QS.q2d_kw(QS.freeform(2, 2, 1e-3, 2), 8.0))
        lens.surfaces.add(index=2, radius=-60.0, thickness=5.0, is_stop=True)
        lens.surfaces.add(index=3, radius=40.0, thickness=4.0, material="N-BK7")
        lens.surfaces.add(index=4, radius=-40.0, thickness=40.0)
        lens.surfaces.add(index=5)
        done()
        lens.set_ray_aiming("robust")
        return lens

    be.set_backend("numpy")
    ref = build(be)
    ref.trace(0.0, 1.0, 0.5876, 6, "hexapolar")
    want = np.array(ref.surfaces.y)
    _install(P, eng, be, which)
    lens = build(be)
    calls = len(eng.calls)
    lens.trace(0.0, 1.0, 0.5876, 6, "hexapolar")
    got = be.to_numpy(lens.surfaces.y)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    assert np.nanmax(np.abs(got - want)) <= 1e-9 * 100.0
    assert not any(c and c[0] == "aim" for c in eng.calls[calls:])
    assert "robust ray aiming: Forbes Q-2D surface before the stop" in P.stats(), P.stats()


# ---- the CUDA kernel -------------------------------------------------------------------------------------------

def _np(t):
    return t.double().cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", PLAIN_CASES)
def test_kernel_fp64_and_fp32_vs_reference_fixture(name):
    import torch

    from optiland_b200.trace import RealRays, SurfaceGroup

    c = Case(name)
    r = c.rays
    for dtype in (torch.float64, torch.float32):
        rays = RealRays(r["x"], r["y"], r["z"], r["L"], r["M"], r["N"], r["i"], r["w"], dtype=dtype)
        sg = SurfaceGroup(c.table)
        sg.trace(rays)
        rec = {k: _np(getattr(sg, k)) for k in REC}
        if dtype == torch.float64:
            _check_fp64(c, rec)
            for k in ("x", "y", "z", "L", "M", "N", "i", "opd"):
                assert max_abs_err(_np(getattr(rays, k)), c.out[k]) <= 1e-11 * c.scale, k
        else:
            got, bound = fp32_errors(rec, c.rec), _bounds(name)
            for k, v in got.items():
                assert v <= 3.0 * bound[k] + 1e-9, (k, v, bound[k])


@pytest.mark.gpu
def test_kernel_m0_only_equals_the_qbfs_twin():
    import torch

    from optiland_b200.trace import RealRays, SurfaceGroup

    q2d, twin = Case("forbes_q2d/q2d_m0_only"), Case("forbes_q2d/q2d_m0_qbfs_twin")
    got = {}
    for c in (q2d, twin):
        r = c.rays
        rays = RealRays(r["x"], r["y"], r["z"], r["L"], r["M"], r["N"], r["i"], r["w"], dtype=torch.float64)
        sg = SurfaceGroup(c.table)
        sg.trace(rays)
        got[id(c)] = {k: _np(getattr(sg, k)) for k in REC}
    for k in REC:
        assert max_abs_err(got[id(q2d)][k], got[id(twin)][k]) <= 1e-11 * twin.scale, k


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
def test_kernel_polarized_fixture_and_intensity_epilogue(dtype_name):
    import torch

    from optiland_b200.trace import PolarizedRays, SurfaceGroup

    dtype = getattr(torch, dtype_name)
    c = Case("forbes_q2d/q2d_polarized")
    r = c.rays
    rays = PolarizedRays(r["x"], r["y"], r["z"], r["L"], r["M"], r["N"], r["i"], r["w"], dtype=dtype)
    sg = SurfaceGroup(c.table)
    sg.trace(rays)
    f64 = dtype == torch.float64
    b = _bounds("forbes_q2d/q2d_polarized")
    for k in ("x", "y", "opd", "L", "M", "N"):
        tag = "opd" if k == "opd" else ("dir" if k in "LMN" else "pos")
        if f64:
            assert max_abs_err(_np(getattr(sg, k)), c.rec[k]) <= 1e-11 * c.scale, k
        else:
            assert fp32_errors({q: _np(getattr(sg, q)) for q in REC}, c.rec)[tag] <= 3 * b[tag], k
    p = rays.p.to(torch.complex128).cpu().numpy()
    assert np.nanmax(np.abs(p - c.out["p"])) <= (1e-11 if f64 else 3 * b["p"])
    rays.update_intensity(None)
    want = c.extra("final_intensity_unpolarized")
    got = _np(rays.i)
    m = np.isfinite(want) & np.isfinite(got)
    assert np.mean(np.isfinite(want) != np.isfinite(got)) <= (0 if f64 else 0.02)
    # i = |P E|^2 / 2 summed over two unit states: its error is at most 2 |dP| per state
    assert np.max(np.abs(got[m] - want[m])) <= (1e-11 if f64 else 3 * 2 * b["p"])


@pytest.mark.gpu
def test_host_buffer_entry_point_matches_device_path():
    """olb_trace_host_* (pinned host buffers, chunked) on the Q-2D singlet == the device path, bit for bit."""
    import torch

    from optiland_b200.trace import DeviceTable, RealRays, SurfaceGroup, trace_host

    c = Case("forbes_q2d/q2d_singlet")
    n = 100_003
    idx = np.random.default_rng(3).integers(0, c.n, size=n)
    for dtype, npt in ((torch.float32, np.float32), (torch.float64, np.float64)):
        h_in = {k: torch.from_numpy(c.rays[k][idx].astype(npt)).pin_memory() for k in c.rays}
        h_out = {k: torch.empty(n, dtype=dtype).pin_memory() for k in ("x", "y", "z", "L", "M", "N", "i", "opd")}
        trace_host(DeviceTable(c.table), h_in, h_out, n, dtype, chunk=30_001)
        r = {k: v[idx] for k, v in c.rays.items()}
        rays = RealRays(r["x"], r["y"], r["z"], r["L"], r["M"], r["N"], r["i"], r["w"], dtype=dtype)
        SurfaceGroup(c.table).trace(rays)
        for k in ("x", "y", "z", "L", "M", "N", "i", "opd"):
            assert np.array_equal(h_out[k].numpy(), getattr(rays, k).cpu().numpy(), equal_nan=True), k


@pytest.mark.gpu
def test_kernel_declines_excluded_mixes_and_aiming():
    """At the C ABI: a Q-2D table with a phase surface is OLB_ERR_UNSUPPORTED at trace time, and so is ray aiming."""
    import torch

    from optiland_b200.trace import RealRays, SurfaceGroup

    doe = T.SurfaceSpec(kind=T.GEOM_PLANE, t=[0, 0, 3.0], interaction=T.INTERACT_PHASE_RADIAL, phase_terms=[-1.0])
    tab = _table(_q2d(), doe)
    rays = RealRays(np.zeros(4), np.zeros(4), np.zeros(4), np.zeros(4), np.zeros(4), np.ones(4), np.ones(4),
                    np.full(4, 0.55), dtype=torch.float64)
    with pytest.raises(Exception, match="Q-2D"):
        SurfaceGroup(tab).trace(rays)
