"""Thin-film, polarizer and retarder coatings (Optiland's ``ThinFilmCoating``, ``PolarizerCoating`` and
``RetarderCoating``) on the polarized trace path: the C ABI and table layer, the per-ray thin-film arithmetic against
the reference's transfer-matrix method, and live reference systems traced through the plugin against the reference's
own NumPy trace.  GPU tests are marked; the rest runs on the CPU through the host instantiation of the kernel variant
of these tables (tests/hostcheck/hostcheck_coating.cpp) and the test engine built on it (oracle/coating_engines.py)."""
import ctypes as C

import numpy as np
import pytest

from oracle import ref_import as pytest_ref
from optiland_b200 import table as T

FEAT_POL, FEAT_JONES = 1 << 3, 1 << 7
needs_ref = pytest.mark.skipif(not pytest_ref.reference_available(), reason="reference not present on this box")
LIVE_REC = ("x", "y", "z", "L", "M", "N", "opd", "intensity")
SYSTEMS = ["coated_doublet", "qwot_singlet", "absorbing_fold", "zero_layer", "polarizer_nested", "retarders",
           "polarizer_refracting", "mixed", "film_on_doe_and_grating"]


def _film(L=2, n_wl=1, **kw):
    d = kw.pop("d", np.linspace(0.08, 0.12, L))
    return dict(coating=T.COAT_THIN_FILM, film_thickness=d, film_n=np.full((L, n_wl), 1.38) + np.arange(L)[:, None],
                film_k=np.zeros((L, n_wl)), film_n0=np.ones(n_wl), film_k0=np.zeros(n_wl), film_ns=np.full(n_wl, 1.5),
                film_ks=np.zeros(n_wl), **kw)


def _table(*coats, n_wl=1, wl=None):
    wl = [0.55, 0.65, 0.45][:n_wl] if wl is None else wl
    specs = [T.SurfaceSpec(kind=T.GEOM_NOOP, n1=np.ones(n_wl), n2=np.ones(n_wl), k1=np.zeros(n_wl))]
    for j, c in enumerate(coats):
        specs.append(T.SurfaceSpec(kind=T.GEOM_STANDARD, radius=40.0, t=[0, 0, 2.0 * j], n1=np.ones(n_wl),
                                   n2=np.full(n_wl, 1.5), k1=np.zeros(n_wl), **c))
    return T.SurfaceTable(specs, wl)


# ---- ABI / table layer -----------------------------------------------------------------------------------------

def test_coating_blocks_pack_after_the_media_block_and_round_trip():
    tab = _table(_film(L=3, n_wl=2), dict(coating=T.COAT_POLARIZER, jones_axis=[0.6, 0.8, 0.0]),
                 dict(coating=T.COAT_RETARDER, retardance=np.pi / 2, jones_axis=[0.0, 1.0, 0.0]), _film(L=0, n_wl=2),
                 n_wl=2)
    surf, pool = tab.pack()
    assert list(surf["coating"]) == [0, 3, 4, 5, 3]
    m = surf["media_off"]
    assert pool[m[1] + 10] == 3.0 and list(pool[m[1] + 11:m[1] + 14]) == list(tab.surfaces[1].film_thickness)
    assert list(pool[m[2] + 10:m[2] + 13]) == [0.6, 0.8, 0.0]
    assert list(pool[m[3] + 10:m[3] + 14]) == [np.pi / 2, 0.0, 1.0, 0.0]
    back = T.SurfaceTable.unpack(surf, pool, tab.wavelengths)
    for a, b in zip(tab.surfaces, back.surfaces):
        assert a.coating == b.coating
        np.testing.assert_array_equal(a.coating_block(), b.coating_block())
    assert back.content_key() == tab.content_key()
    for bad in (dict(d=[np.nan, 0.1]), dict(d=[-0.1, 0.1])):
        with pytest.raises(ValueError, match="thin film"):
            _table(_film(**bad))
    with pytest.raises(ValueError, match="thin film"):
        _table(_film(L=T.MAX_FILM_LAYERS + 1))
    # the prepared records of a table are capped (they are staged in shared memory): 32 layers at 16 wavelengths on
    # 3 surfaces fit, on 4 they do not
    with pytest.raises(ValueError, match="shared memory"):
        _table(*[_film(L=32, n_wl=16)] * 4, n_wl=16, wl=list(np.linspace(0.45, 0.7, 16)))
    _table(*[_film(L=32, n_wl=16)] * 3, n_wl=16, wl=list(np.linspace(0.45, 0.7, 16)))
    for axis in ([0, 0, 0], [np.nan, 1, 0]):
        with pytest.raises(ValueError, match="axis"):
            _table(dict(coating=T.COAT_POLARIZER, jones_axis=axis))


def test_uncoated_table_packs_as_before():
    """A table without these coatings packs byte for byte as without the coating fields."""
    tab = _table(dict(), dict(coating=T.COAT_FRESNEL, coat_n1=[1.0], coat_n2=[1.5]))
    surf, pool = tab.pack()
    want = [1.0, 1.0, 0.0, 1.0, 1.0, 0.0] + [1.0, 1.5, 0.0, 1.0, 1.5, 0.0] * 2   # media blocks, each padded to even
    assert list(pool) == want and list(surf["media_off"]) == [0, 6, 12]


def _raw(tab, mutate):
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


def test_upload_errors_and_feature_bits():
    film = _table(_film(L=2))
    rc, msg, feat = _raw(film, lambda s, p: None)
    assert rc > 0 and feat & FEAT_POL and feat & FEAT_JONES
    pol = _table(dict(coating=T.COAT_POLARIZER, jones_axis=[1.0, 0.0, 0.0]))
    ret = _table(dict(coating=T.COAT_RETARDER, retardance=1.0, jones_axis=[1.0, 0.0, 0.0]))
    for t in (pol, ret):
        rc, msg, feat = _raw(t, lambda s, p: None)
        assert rc > 0 and feat & FEAT_JONES

    def cb(s):
        return s["media_off"][1] + 5

    def layers_high(s, p):
        p[cb(s)] = T.MAX_FILM_LAYERS + 1

    def layers_frac(s, p):
        p[cb(s)] = 1.5

    def thickness(s, p):
        p[cb(s) + 1] = -1.0

    def outside(s, p):
        s["media_off"][1] = len(p) - 5

    def on_object(s, p):
        s["coating"][0] = T.COAT_THIN_FILM

    def unknown(s, p):
        s["coating"][1] = 6

    for mutate, word in ((layers_high, "layers"), (layers_frac, "layers"), (thickness, "thickness"),
                         (outside, "outside"), (on_object, "object"), (unknown, "unknown coating")):
        rc, msg, feat = _raw(film, mutate)
        assert rc == -5 and word in msg and feat == -1, (mutate.__name__, rc, msg)

    def zero_axis(s, p):
        p[cb(s):cb(s) + 3] = 0.0

    rc, msg, feat = _raw(pol, zero_axis)
    assert rc == -5 and "axis" in msg

    def nan_retardance(s, p):
        p[cb(s)] = np.nan

    rc, msg, feat = _raw(ret, nan_retardance)
    assert rc == -5 and "retardance" in msg


def test_backward_and_batched_uploads_refuse_coated_tables():
    from optiland_b200 import _lib
    from optiland_b200.batch import template_params
    from oracle.hostcheck_api import load

    tab = _table(_film(L=1))
    ht = _lib.HostTable(tab)
    hc = load()
    assert hc.olbhc_bwd_supported(C.byref(ht.c)) == 0
    params = np.zeros((2, tab.num_surfaces, _lib.BP_COUNT))
    lib = _lib.load()
    ws = np.zeros(1 << 16, dtype=np.uint8)
    dt = _lib.OlbDeviceTable()
    rc = lib.olb_table_upload_batch(C.byref(ht.c), C.c_void_p(params.ctypes.data), 2,
                                    C.c_void_p((ws.ctypes.data + 15) & ~15), C.c_int64(ws.size - 16), None, C.byref(dt))
    assert rc == -2
    with pytest.raises(ValueError, match="thin-film"):
        template_params(tab)


# ---- per-ray thin-film arithmetic vs the reference's transfer-matrix method -----------------------------------------

@needs_ref
@pytest.mark.parametrize("absorbing", [False, True])
def test_thin_film_rt_matches_reference_tmm(absorbing):
    """r and t of the host arithmetic against ThinFilmStack.compute_rtRTA_elementwise, for s and p, over angles of
    incidence from 0 to near grazing and three wavelengths, with and without absorbing layers."""
    pytest_ref.import_reference()
    import optiland.backend as be
    from optiland.materials import IdealMaterial
    from optiland.thin_film import ThinFilmStack

    from oracle.hostcheck_coating import film_rt

    be.set_backend("numpy")
    k = 0.4 if absorbing else 0.0
    mats = [IdealMaterial(n=1.38), IdealMaterial(n=2.35, k=k), IdealMaterial(n=1.46), IdealMaterial(n=2.0, k=k / 2)]
    thick = [0.1, 0.06, 0.35, 0.02]
    stack = ThinFilmStack(IdealMaterial(n=1.0), IdealMaterial(n=1.52, k=0.01 if absorbing else 0.0))
    for m, d in zip(mats, thick):
        stack.add_layer(m, d)
    wls = np.array([0.45, 0.55, 0.7])
    spec = dict(coating=T.COAT_THIN_FILM, film_thickness=thick,
                film_n=np.array([[m.n(w) for w in wls] for m in mats]).reshape(4, 3),
                film_k=np.array([[m.k(w) for w in wls] for m in mats]).reshape(4, 3),
                film_n0=np.ones(3), film_k0=np.zeros(3), film_ns=np.full(3, 1.52),
                film_ks=np.full(3, 0.01 if absorbing else 0.0))
    tab = _table(spec, n_wl=3, wl=wls)
    aoi = np.concatenate([np.linspace(0.0, 1.5, 31), [1.55, 1.565]])
    A, W = np.meshgrid(aoi, np.arange(3))
    A, W = A.ravel(), W.ravel()
    rs, ts, rp, tp = film_rt(tab, 1, W, A)
    rs32, ts32, rp32, tp32 = film_rt(tab, 1, W, A, np.float32)
    for pol, (r, t), (r32, t32) in (("s", (rs, ts), (rs32, ts32)), ("p", (rp, tp), (rp32, tp32))):
        want = stack.compute_rtRTA_elementwise(wls[W], A, pol)
        for got, got32, ref in ((r, r32, want["r"]), (t, t32, want["t"])):
            err = np.abs(got - ref) / np.maximum(np.abs(ref), 1e-3)
            assert np.max(err) <= 1e-12, (pol, float(np.max(err)))
            # fp32, up to 89.7 degrees: the incident medium's term is formed from cos^2, so it does not cancel near
            # grazing (measured: below 2e-6)
            assert np.max(np.abs(got32 - ref)) <= 1e-5, (pol, "fp32", float(np.max(np.abs(got32 - ref))))


# ---- live reference systems through the plugin --------------------------------------------------------------------

@pytest.fixture(params=["devmath", pytest.param("cuda", marks=pytest.mark.gpu)])
def live(request):
    pytest_ref.import_reference()
    import optiland.backend as be

    from optiland_b200 import plugin as P

    if request.param == "cuda":
        eng = P.CudaEngine()
    else:
        from oracle.coating_engines import CoatingDeviceMathEngine

        eng = CoatingDeviceMathEngine()
    yield P, eng, be, request.param
    if P._state.get("installed"):
        P.uninstall()
    if request.param == "cuda":
        be.set_device("cpu")
    be.set_backend("numpy")


def _install(P, eng, be, which, precision="float64"):
    be.set_backend("torch")
    be.set_precision(precision)
    be.grad_mode.disable()
    if which == "cuda":
        be.set_device("cuda")
    P.install(engine=eng)
    P.stats(reset=True)


def _close(got, want, tol, what):
    assert got.shape == want.shape, what
    assert np.array_equal(np.isnan(got), np.isnan(want)), (what, "NaN pattern")
    m = np.isfinite(want)
    assert not m.any() or np.max(np.abs(got[m] - want[m])) <= tol, (what, float(np.max(np.abs(got[m] - want[m]))))


def _reference_runs(system, be):
    from tests import _coating_systems as CS

    be.set_backend("numpy")
    ref = CS.BUILDERS[system](be)
    wls = [float(w.value) for w in ref.wavelengths.wavelengths]
    jobs = [(hy, wl) for hy in (0.0, 1.0) for wl in wls]
    want = []
    for hy, wl in jobs:
        r = ref.trace(0.0, hy, wl, 10, "hexapolar")
        want.append(({k: np.array(getattr(ref.surfaces, k)) for k in LIVE_REC},
                     {"i": np.array(r.i), "p": np.array(r.p)}))
    return jobs, want


@needs_ref
@pytest.mark.parametrize("system", SYSTEMS)
def test_optic_trace_through_the_plugin_equals_the_reference(live, system):
    """Optic.trace of every field x wavelength: each record row, the final polarized intensity and rays.p equal the
    NumPy reference, in one fused launch per trace, no decline."""
    from tests import _coating_systems as CS

    P, eng, be, which = live
    jobs, want = _reference_runs(system, be)
    _install(P, eng, be, which)
    lens = CS.BUILDERS[system](be)
    n0 = len(eng.calls)
    for (hy, wl), (w, wr) in zip(jobs, want):
        r = lens.trace(0.0, hy, wl, 10, "hexapolar")
        scale = max(1.0, float(np.nanmax(np.abs(w["z"]))))
        for k, v in w.items():
            _close(be.to_numpy(getattr(lens.surfaces, k)), v, 1e-11 * scale, k)
        _close(be.to_numpy(r.i), wr["i"], 1e-12, "i")
        _close(be.to_numpy(r.p), wr["p"], 1e-12, "p")
    assert not P.stats(), P.stats()
    assert sum(1 for c in eng.calls[n0:] if c and c[0] == "pupil") == len(jobs), eng.calls[n0:]


@needs_ref
def test_trace_generic_and_analyses_on_the_coated_doublet(live):
    """trace_generic with a linear polarized state, the polarized Wavefront and the Jones pupil (JonesPupil, every
    wavelength) on the coated doublet equal the reference."""
    from tests import _coating_systems as CS

    P, eng, be, which = live
    be.set_backend("numpy")
    ref = CS.coated_doublet(be, polarized=True)
    from optiland.wavefront import Wavefront

    Px, Py = np.linspace(-0.9, 0.9, 7), np.linspace(0.8, -0.8, 7)
    rg = ref.trace_generic(Hx=0.0, Hy=0.7, Px=Px, Py=Py, wavelength=0.5876)
    want_g = {k: np.array(getattr(rg, k)) for k in ("x", "y", "L", "M", "N", "i", "opd")}
    wf = Wavefront(ref, fields=[(0.0, 1.0)], wavelengths=[0.5876], num_rays=8, distribution="hexapolar")
    want_w = {k: np.array(getattr(wf.data[((0.0, 1.0), 0.5876)], k)) for k in ("opd", "intensity")}
    from optiland.analysis import JonesPupil

    # JonesPupil stores J in a real tensor on the torch backend (the reference drops the imaginary part there), so the
    # plugin's result is compared with the real part of the NumPy reference's J
    want_j = [np.array(d["J"]).real for d in JonesPupil(ref, field=(0.0, 1.0), grid_size=9).data]
    _install(P, eng, be, which)
    lens = CS.coated_doublet(be, polarized=True)
    g = lens.trace_generic(Hx=0.0, Hy=0.7, Px=be.array(Px), Py=be.array(Py), wavelength=0.5876)
    for k, v in want_g.items():
        _close(be.to_numpy(getattr(g, k)), v, 1e-10, k)
    wf = Wavefront(lens, fields=[(0.0, 1.0)], wavelengths=[0.5876], num_rays=8, distribution="hexapolar")
    for k, v in want_w.items():
        _close(be.to_numpy(getattr(wf.data[((0.0, 1.0), 0.5876)], k)), v, 1e-9, k)
    got_j = [be.to_numpy(d["J"]) for d in JonesPupil(lens, field=(0.0, 1.0), grid_size=9).data]
    assert len(got_j) == len(want_j) == 3
    for g, w in zip(got_j, want_j):
        _close(g, w, 1e-11, "Jones pupil")
    assert not P.stats(), P.stats()


@needs_ref
def test_declined_coating_configurations():
    """A subclass of a coating class, a stack of more than OLB_MAX_FILM_LAYERS layers and gradients wanted each
    decline to the reference with their reason."""
    pytest_ref.import_reference()
    import optiland.backend as be
    from optiland.coatings import ThinFilmCoating
    from optiland.materials import IdealMaterial

    from optiland_b200 import plugin as P
    from oracle.coating_engines import CoatingDeviceMathEngine
    from tests import _coating_systems as CS

    class MyFilm(ThinFilmCoating):
        pass

    try:
        _install(P, CoatingDeviceMathEngine(), be, "devmath")
        for coating, word in ((MyFilm(IdealMaterial(n=1.0), IdealMaterial(n=1.5), [(IdealMaterial(n=1.38), 100.0, "a")]),
                               "coating MyFilm"),
                              (ThinFilmCoating(IdealMaterial(n=1.0), IdealMaterial(n=1.5),
                                               [(IdealMaterial(n=1.38 + 0.5 * (i % 2)), 50.0, str(i)) for i in range(33)]),
                               "more than 32 layers")):
            lens = CS.zero_layer(be)
            lens.surfaces.surfaces[1].interaction_model.coating = coating
            P.stats(reset=True)
            lens.trace(0.0, 0.0, 0.5876, 4, "hexapolar")
            assert any(word in k for k in P.stats()), P.stats()
        be.grad_mode.enable()
        lens = CS.zero_layer(be)
        P.stats(reset=True)
        lens.trace(0.0, 0.0, 0.5876, 4, "hexapolar")
        assert any("gradients wanted" in k for k in P.stats()), P.stats()
    finally:
        be.grad_mode.disable()
        P.uninstall()
        be.set_backend("numpy")


# ---- known answers -------------------------------------------------------------------------------------------------

# (axis, Jones block (J00, J01, J10, J11)) of the reference's tests/test_jones.py: JonesPolarizerH / V / L45 / L135
KNOWN_POLARIZERS = [((1.0, 0.0, 0.0), (1.0, 0.0, 0.0, 0.0)), ((0.0, 1.0, 0.0), (0.0, 0.0, 0.0, 1.0)),
                    ((1.0, 1.0, 0.0), (0.5, 0.5, 0.5, 0.5)), ((-1.0, 1.0, 0.0), (0.5, -0.5, -0.5, 0.5))]


@pytest.mark.parametrize("engine", ["devmath", pytest.param("cuda", marks=pytest.mark.gpu)])
@pytest.mark.parametrize("axis,want", KNOWN_POLARIZERS)
def test_known_answers_of_the_reference_jones_tests(engine, axis, want):
    """A polarizer on a plane at normal incidence: the basis is s = x, p0 = p1 = y (the k0 || k1 fallback of
    get_local_basis), so the traced P matrix of an identity input is the Jones block itself, and it equals the values
    the reference's own polarizer tests pin."""
    import torch

    a = np.asarray(axis) / np.linalg.norm(axis)    # normalised once, as JonesLinearPolarizer does
    tab = T.SurfaceTable([T.SurfaceSpec(kind=T.GEOM_NOOP),
                          T.SurfaceSpec(kind=T.GEOM_PLANE, t=[0, 0, 1.0], coating=T.COAT_POLARIZER, jones_axis=a)], [0.55])
    n = 3
    rays = dict(x=np.array([0.0, 0.5, -1.0]), y=np.array([0.0, 0.2, 0.3]), z=np.zeros(n), L=np.zeros(n), M=np.zeros(n),
                N=np.ones(n), i=np.ones(n), w=np.full(n, 0.55), opd=np.zeros(n))
    pm = np.tile(np.eye(3, dtype=np.complex128), (n, 1, 1))
    if engine == "cuda":
        from optiland_b200.trace import PolarizedRays, SurfaceGroup

        sg = SurfaceGroup(tab, device="cuda:0")
        pr = PolarizedRays(*(torch.tensor(rays[k]) for k in ("x", "y", "z", "L", "M", "N", "i", "w")),
                           dtype=torch.float64, device="cuda:0")
        sg.trace(pr)
        P = pr.p.cpu().numpy()
    else:
        from oracle.hostcheck_coating import run_hostcheck_coating

        P = run_hostcheck_coating(tab, rays, np.float64, pmat=pm)[0]["p"]
    J = np.stack([P[:, 0, 0], P[:, 0, 1], P[:, 1, 0], P[:, 1, 1]], axis=1)
    np.testing.assert_allclose(J, np.tile(np.asarray(want, dtype=complex), (n, 1)), atol=1e-15)
    np.testing.assert_allclose(P[:, 2, 2], 1.0, atol=1e-15)


@needs_ref
@pytest.mark.gpu
@pytest.mark.timeout(1500)
@pytest.mark.parametrize("fname", ["test_coatings.py", "test_jones.py"])
def test_reference_coating_and_jones_tests_unchanged_with_cuda_engine(fname):
    """The reference's own tests/test_coatings.py and tests/test_jones.py with the torch backend on the GPU, stock vs.
    the plugin over the product CudaEngine: the same failing set.  (These tests call the coatings' and Jones classes'
    own methods on hand-built rays, not SurfaceGroup.trace, so the plugin is installed without being asked to trace;
    the known answers they pin for the polarizers are asserted through the kernel above.)"""
    from tests.test_reference_sweep import _run

    stock, _, bad_stock, _ = _run(fname, install=False, nograd=True, cuda=True, with_ids=True)
    ours, _, bad_ours, _ = _run(fname, install=True, nograd=True, cuda=True, with_ids=True)
    print(f"{fname}: stock {stock} | plugin {ours}")
    assert stock.get("passed", 0) > 0, stock
    assert bad_ours == bad_stock and ours == stock, (stock, ours, bad_stock, bad_ours)


# ---- fp32 on the GPU -------------------------------------------------------------------------------------------------

@needs_ref
@pytest.mark.gpu
@pytest.mark.parametrize("system", SYSTEMS)
def test_kernel_fp32_against_reference(system):
    """The fp32 kernel through the plugin against the fp64 NumPy reference: positions within 1.5e-5 x system scale,
    the polarized intensity and rays.p within 3e-5, about three times the largest errors measured on an H100 (4.8e-6
    x scale, 9.3e-6 in i and 4.6e-6 in p, all on the quarter-wave singlet)."""
    pytest_ref.import_reference()
    import optiland.backend as be

    from optiland_b200 import plugin as P
    from tests import _coating_systems as CS

    jobs, want = _reference_runs(system, be)
    try:
        _install(P, P.CudaEngine(), be, "cuda", precision="float32")
        lens = CS.BUILDERS[system](be)
        worst = {"pos": 0.0, "i": 0.0, "p": 0.0}
        for (hy, wl), (w, wr) in zip(jobs, want):
            r = lens.trace(0.0, hy, wl, 10, "hexapolar")
            scale = max(1.0, float(np.nanmax(np.abs(w["z"]))))
            for k in ("x", "y", "z"):
                g = be.to_numpy(getattr(lens.surfaces, k)).astype(np.float64)
                assert np.array_equal(np.isnan(g), np.isnan(w[k])), (k, "NaN pattern")
                m = np.isfinite(w[k])
                worst["pos"] = max(worst["pos"], float(np.max(np.abs(g[m] - w[k][m]), initial=0)) / scale)
            for k in ("i", "p"):
                g = be.to_numpy(getattr(r, k))
                assert np.array_equal(np.isnan(g), np.isnan(wr[k])), (k, "NaN pattern")
                m = np.isfinite(wr[k])
                worst[k] = max(worst[k], float(np.max(np.abs(g[m] - wr[k][m]), initial=0)))
        print(system, "fp32 worst", worst)
        assert not P.stats(), P.stats()
        assert worst["pos"] <= 1.5e-5 and worst["i"] <= 3e-5 and worst["p"] <= 3e-5, worst
    finally:
        P.uninstall()
        be.set_device("cpu")
        be.set_precision("float64")
        be.set_backend("numpy")
