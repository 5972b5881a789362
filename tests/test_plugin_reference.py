"""The Optiland plugin (backend registration, RealRayTracer / SurfaceGroup.trace / Surface.trace wrappers, packing of
LIVE reference objects, record hand-back, autograd, declining) exercised against the unmodified reference: the build
copy of the reference that build() stages under oracle/_ref/ (oracle/make_ref.sh).

Every test runs twice:
* ``[oracle]`` (CPU, ``-m "not gpu"``): there is no GPU in the build container, so the device call is replaced by a
  TEST-ONLY engine that evaluates the packed table with the NumPy oracle; everything else is the product code path;
* ``[cuda]`` (``-m gpu``, on the GPU): the PRODUCT engine (``plugin.CudaEngine`` -> libolb.so) under
  ``be.set_device("cuda")`` with live Optiland objects -- ``Optic.trace``, ``SpotDiagram``, ``Wavefront``, the
  optimiser's autograd step and the aimers call the CUDA kernels unchanged, compared with the reference's NumPy path.
"""
import numpy as np
import pytest

from oracle.ref_import import reference_available

pytestmark = pytest.mark.skipif(not reference_available(), reason="reference not present on this box")


from oracle.oracle_engine import OracleEngine  # noqa: E402


@pytest.fixture(params=["oracle", pytest.param("cuda", marks=pytest.mark.gpu)])
def plugin(request):
    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be

    from optiland_b200 import _lib
    from optiland_b200 import plugin as P

    be.set_backend("torch")
    be.set_precision("float64")
    be.grad_mode.disable()
    launches0 = 0
    if request.param == "cuda":
        be.set_device("cuda")
        eng = P.CudaEngine()
        launches0 = _lib.load().olb_launch_count()
    else:
        eng = OracleEngine()
    P.install(engine=eng)
    P.stats(reset=True)
    yield P, eng, be
    if request.param == "cuda":
        # the calls the test counted really were kernel launches of libolb.so
        assert not eng.calls or _lib.load().olb_launch_count() > launches0
        be.set_device("cpu")
    P.uninstall()
    be.set_backend("numpy")


def _numpy_reference(make_lens, trace):
    import optiland.backend as be

    be.set_backend("numpy")
    lens = make_lens()
    rays = trace(lens)
    out = {k: np.array(getattr(lens.surfaces, k)) for k in ("x", "y", "z", "L", "M", "N", "opd", "intensity")}
    fin = {k: np.array(getattr(rays, k)) for k in ("x", "y", "z", "L", "M", "N", "i", "opd")}
    be.set_backend("torch")
    return out, fin


def test_backend_registration_keeps_name_torch(plugin):
    P, eng, be = plugin
    assert be.get_backend() == "torch"
    backend = be.__getattr__.__globals__["_backends"]["torch"]
    assert type(backend).__name__ == "B200TorchBackend" and backend.name == "torch"
    assert hasattr(backend, "trace_surfaces")
    assert float(be.sin(be.array(0.5))) == pytest.approx(np.sin(0.5))  # every TorchBackend op still there


def test_optic_trace_goes_through_capability_and_matches_numpy(plugin):
    P, eng, be = plugin
    from optiland.samples.objectives import DoubleGauss

    def trace(lens):
        return lens.trace(Hx=0.0, Hy=0.7, wavelength=0.5876, num_rays=8, distribution="hexapolar")

    ref_rec, ref_fin = _numpy_reference(DoubleGauss, trace)
    lens = DoubleGauss()
    rays = trace(lens)
    assert eng.calls and eng.calls[-1][:2] == ("pupil", 13)  # Optic.trace: launch generated in the engine call
    for k, v in ref_rec.items():
        got = be.to_numpy(getattr(lens.surfaces, k))
        assert got.shape == v.shape
        np.testing.assert_allclose(got, v, rtol=0, atol=1e-11)
    for k, v in ref_fin.items():
        np.testing.assert_allclose(be.to_numpy(getattr(rays, k)), v, rtol=0, atol=1e-11)
    # L0/M0/N0 = direction before the last interaction
    np.testing.assert_allclose(be.to_numpy(rays.L0), ref_rec["L"][-2], atol=1e-12)


def test_optic_trace_fused_launch_for_finite_and_telecentric_objects(plugin):
    """f-1 beyond infinite-object angle fields: object-height field on a finite object, and the
    object-space telecentric 44-surface lithography sample -- Optic.trace goes through the fused launch
    and reproduces the NumPy reference, record by record."""
    P, eng, be = plugin
    from optiland.samples.lithography import UVProjectionLens

    from oracle.make_golden import finite_relay

    for make, H, wl, S in ((lambda: finite_relay("object_height"), (2.0 / 9.0, 1.0), 0.5876, 5),
                           (lambda: finite_relay("angle"), (0.25, 1.0), 0.5876, 5),
                           (UVProjectionLens, (0.0, 1.0), 0.248, 44)):
        def trace(lens):
            return lens.trace(Hx=H[0], Hy=H[1], wavelength=wl, num_rays=6, distribution="hexapolar")

        ref_rec, ref_fin = _numpy_reference(make, trace)
        lens = make()
        rays = trace(lens)
        assert eng.calls[-1][:2] == ("pupil", S), eng.calls[-1]
        scale = max(1.0, float(np.nanmax(np.abs(ref_rec["z"]))))
        for k, v in ref_rec.items():
            got = be.to_numpy(getattr(lens.surfaces, k))
            assert got.shape == v.shape
            np.testing.assert_allclose(got, v, rtol=0, atol=1e-11 * scale, err_msg=k)
        for k, v in ref_fin.items():
            np.testing.assert_allclose(be.to_numpy(getattr(rays, k)), v, rtol=0, atol=1e-11 * scale, err_msg=k)


def test_trace_generic_with_per_ray_fields_and_wavelengths(plugin):
    """trace_generic (config 5's call shape: per-ray Hx, Hy, Px, Py and wavelength arrays) goes through the fused
    launch with per-ray field points and reproduces the NumPy reference; a system with vignetting factors declines."""
    P, eng, be = plugin
    from optiland.samples.objectives import DoubleGauss
    from optiland.samples.lithography import UVProjectionLens

    from oracle.make_golden import finite_relay

    rng = np.random.default_rng(3)
    n = 60
    Px, Py = rng.uniform(-0.7, 0.7, n), rng.uniform(-0.7, 0.7, n)
    Hx, Hy = rng.uniform(-0.5, 0.5, n), rng.uniform(-0.8, 0.8, n)
    for make, wls, S in ((DoubleGauss, [0.4861, 0.5876, 0.6563], 13), (lambda: finite_relay("object_height"), [0.5876], 5),
                         (UVProjectionLens, [0.248], 44)):
        wl = np.asarray(wls)[rng.integers(0, len(wls), n)]

        def trace(lens):
            a = lambda v: be.array(v)  # noqa: E731
            return lens.trace_generic(a(Hx), a(Hy), a(Px), a(Py), a(wl) if len(wls) > 1 else float(wls[0]))

        ref_rec, ref_fin = _numpy_reference(make, trace)
        lens = make()
        n0 = len(eng.calls)
        rays = trace(lens)
        assert ("pupil", S, n) in [c[:3] for c in eng.calls[n0:]], (eng.calls[n0:], P.stats())
        scale = max(1.0, float(np.nanmax(np.abs(ref_rec["z"]))))
        for k, v in ref_rec.items():
            np.testing.assert_allclose(be.to_numpy(getattr(lens.surfaces, k)), v, rtol=0, atol=1e-11 * scale, err_msg=k)
        for k, v in ref_fin.items():
            np.testing.assert_allclose(be.to_numpy(getattr(rays, k)), v, rtol=0, atol=1e-11 * scale, err_msg=k)
    # vignetting factors (nearest-neighbour per ray, applied twice on this path by the reference): reproduced
    def make_vig():
        lens = DoubleGauss()
        lens.fields.fields[1].vy = 0.1
        lens.fields.fields[2].vx = 0.05
        return lens

    def trace_v(lens):
        a = lambda v: be.array(v)  # noqa: E731
        return lens.trace_generic(a(Hx), a(Hy), a(Px), a(Py), 0.5876)

    ref_rec, ref_fin = _numpy_reference(make_vig, trace_v)
    lens = make_vig()
    n0 = len(eng.calls)
    rays = trace_v(lens)
    assert ("pupil", 13, n) in [c[:3] for c in eng.calls[n0:]]
    for k, v in ref_rec.items():
        np.testing.assert_allclose(be.to_numpy(getattr(lens.surfaces, k)), v, rtol=0, atol=1e-10, err_msg=k)
    assert float(np.max(np.abs(ref_rec["x"][1] - np.asarray(_numpy_reference(DoubleGauss, trace_v)[0]["x"][1])))) > 1e-3


def test_wavefront_analysis_uses_the_fused_epilogue(plugin):
    """f-2: Wavefront(strategy='chief_ray') under the plugin == the NumPy reference, and the full-grid trace
    went through the wavefront capability (5 values per ray, no records)."""
    P, eng, be = plugin
    from optiland.samples.objectives import CookeTriplet
    from optiland.wavefront import Wavefront

    from oracle.make_golden import finite_relay

    for make, field, wl in ((CookeTriplet, (0.0, 0.7), 0.55), (lambda: finite_relay("object_height"), (0.0, 1.0), 0.5876)):
        def run(lens):
            w = Wavefront(lens, fields=[field], wavelengths=[wl], num_rays=8, distribution="hexapolar", strategy="chief_ray")
            d = w.get_data(field, wl)
            return {k: np.array(be.to_numpy(getattr(d, k)), dtype=np.float64) for k in ("opd", "pupil_x", "pupil_y", "pupil_z", "intensity")}, \
                float(np.asarray(be.to_numpy(d.radius)).reshape(-1)[0])

        be.set_backend("numpy")
        want, Rw = run(make())
        be.set_backend("torch")
        n0 = len(eng.calls)
        got, Rg = run(make())
        assert any(c[0] == "wavefront" for c in eng.calls[n0:]), eng.calls[n0:]
        assert Rg == pytest.approx(Rw, rel=1e-12)
        for k in want:
            np.testing.assert_allclose(got[k], want[k], rtol=0, atol=1e-6 if k == "opd" else 1e-10, err_msg=k)
    # the reference path is still there when the fusion is switched off
    P._state["fuse_wavefront"] = False
    try:
        n0 = len(eng.calls)
        lens = CookeTriplet()
        Wavefront(lens, fields=[(0.0, 0.7)], wavelengths=[0.55], num_rays=6, distribution="hexapolar", strategy="chief_ray")
        assert not any(c[0] == "wavefront" for c in eng.calls[n0:])
    finally:
        P._state["fuse_wavefront"] = True


def test_spot_diagram_runs_unchanged_on_top(plugin):
    """Config 1: analysis layer untouched; golden RMS radii of the reference's tests/test_analysis.py:88-102."""
    P, eng, be = plugin
    from optiland.analysis import SpotDiagram
    from optiland.samples.objectives import CookeTriplet

    spot = SpotDiagram(CookeTriplet())
    rms = spot.rms_spot_radius()
    assert len(eng.calls) >= 9
    golden = [[0.003791335461448, 0.004293689564257, 0.006195618755672],
              [0.01582480029344623, 0.016918412809703662, 0.019221165873836682],
              [0.013236232767092956, 0.012116688566406967, 0.013648684944411313]]
    for f in range(3):
        for w in range(3):
            assert float(rms[f][w]) == pytest.approx(golden[f][w], rel=1e-9)


def test_spot_statistics_from_the_moments_epilogue(plugin):
    """f-2 wired in: SpotDiagram.rms_spot_radius / centroid and the rms_spot_size operand are served by moment launches
    (no per-ray output); the per-ray spot data appears only when something reads it."""
    P, eng, be = plugin
    from optiland.analysis import SpotDiagram
    from optiland.optimization.operand.ray import RayOperand
    from optiland.samples.objectives import CookeTriplet
    from optiland.samples.telescopes import HubbleTelescope

    golden = [[0.003791335461448, 0.004293689564257, 0.006195618755672],
              [0.01582480029344623, 0.016918412809703662, 0.019221165873836682],
              [0.013236232767092956, 0.012116688566406967, 0.013648684944411313]]
    for reference in ("chief_ray", "centroid"):
        be.set_backend("numpy")
        ref_spot = SpotDiagram(CookeTriplet(), reference=reference)
        want = np.array(ref_spot.rms_spot_radius(), dtype=np.float64)
        want_c = np.array(ref_spot.centroid(), dtype=np.float64)
        be.set_backend("torch")
        n0 = len(eng.calls)
        spot = SpotDiagram(CookeTriplet(), reference=reference)
        rms = spot.rms_spot_radius()
        cen = spot.centroid()
        kinds = [c[0] for c in eng.calls[n0:]]
        assert kinds.count("moments") >= 9
        assert not any(c[0] == "pupil" and c[2] > 1 for c in eng.calls[n0:])      # no full-grid records were traced
        got = np.array([[float(v) for v in row] for row in rms])
        np.testing.assert_allclose(got, want, rtol=1e-9)
        np.testing.assert_allclose(np.array([[float(v) for v in c] for c in cen]), want_c, rtol=0, atol=1e-10)
        if reference == "chief_ray":
            np.testing.assert_allclose(got, np.array(golden), rtol=1e-9)          # tests/test_analysis.py:88-102
        # reading the data materialises it: one record launch per spot, same numbers as the reference's eager arrays
        geo = spot.geometric_spot_radius()
        be.set_backend("numpy")
        want_geo = np.array(ref_spot.geometric_spot_radius(), dtype=np.float64)
        be.set_backend("torch")
        np.testing.assert_allclose(np.array([[float(v) for v in row] for row in geo]), want_geo, rtol=1e-9)
        assert any(c[0] == "pupil" and c[2] > 1 for c in eng.calls[n0:])
    # the operand: single wavelength and "all", image surface and an inner surface; Hubble has an obscuration
    for make, args in ((CookeTriplet, dict(surface_number=-1, Hx=0.0, Hy=0.7, num_rays=8, wavelength=0.55)),
                       (CookeTriplet, dict(surface_number=4, Hx=0.0, Hy=1.0, num_rays=6, wavelength="all")),
                       (HubbleTelescope, dict(surface_number=-1, Hx=0.0, Hy=1.0, num_rays=8, wavelength=0.55))):
        be.set_backend("numpy")
        want = float(RayOperand.rms_spot_size(make(), distribution="hexapolar", **args))
        be.set_backend("torch")
        n0 = len(eng.calls)
        got = float(RayOperand.rms_spot_size(make(), distribution="hexapolar", **args))
        assert all(c[0] == "moments" for c in eng.calls[n0:]) and len(eng.calls) > n0, eng.calls[n0:]
        assert got == pytest.approx(want, rel=1e-9)
    assert not any("spot moments" in k for k in P.stats()), P.stats()


def test_declines_and_falls_back_to_reference_python(plugin):
    P, eng, be = plugin
    from optiland.samples.objectives import CookeTriplet

    # unsupported interaction model (paraxial thin lens) -> decline, results still those of the reference
    def make():
        from optiland import optic

        lens = optic.Optic()
        lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
        lens.surfaces.add(index=1, surface_type="paraxial", f=50.0, thickness=5.0, is_stop=True)
        lens.surfaces.add(index=2, radius=-80.0, thickness=50.0, material="N-BK7")
        lens.surfaces.add(index=3)
        lens.set_aperture(aperture_type="EPD", value=10.0)
        lens.fields.set_type(field_type="angle")
        lens.fields.add(y=0)
        lens.wavelengths.add(value=0.55, is_primary=True)
        return lens

    def trace(lens):
        return lens.trace(0.0, 0.0, 0.55, 4, "hexapolar")

    ref_rec, _ = _numpy_reference(make, trace)
    n0 = len(eng.calls)
    lens = make()
    P.stats(reset=True)
    trace(lens)
    assert all(c[0] != 4 for c in eng.calls[n0:])  # the 4-surface group was never handed to the engine
    why = P.stats()
    assert any("unsupported" in k and "ThinLens" in k for k in why), why   # and the plugin says why
    np.testing.assert_allclose(be.to_numpy(lens.surfaces.y), ref_rec["y"], atol=1e-10)


def test_per_surface_entry_used_by_ray_aimers(plugin):
    """Iterative ray aiming (rays/ray_aiming/iterative.py): every Broyden iteration re-traces all rays from the first
    surface to the stop with one ``Surface.trace`` call per surface (:339-367).  Under the plugin the subset is ONE
    table and ONE launch (``IterativeRayAimer._trace_subset`` wrapper -> SurfaceGroup capability over [start, stop]);
    with that fusion switched off the per-surface wrapper carries the calls (one-surface tables), as it does for the
    stop-radius strategy (initialization.py:150).  Both equal the NumPy reference."""
    P, eng, be = plugin
    from optiland.samples.objectives import CookeTriplet

    def trace(lens):
        lens.set_ray_aiming("iterative", max_iter=10, tol=1e-9)
        return lens.trace(0.0, 0.7, 0.55, 4, "hexapolar")

    ref_rec, ref_fin = _numpy_reference(CookeTriplet, trace)
    stop = CookeTriplet().surfaces.stop_index
    for fused in (True, False):
        P._state["fuse_aimer"] = fused
        n0 = len(eng.calls)
        lens = CookeTriplet()
        rays = trace(lens)
        sizes = [c[0] for c in eng.calls[n0:] if isinstance(c[0], int)]
        if fused:
            assert sizes.count(stop) >= 2, sizes            # surfaces 1 .. stop in one table, once per aimer iteration
        else:
            assert sizes.count(1) >= 2 * stop and stop not in sizes[:-1], sizes   # single-surface tables
        np.testing.assert_allclose(be.to_numpy(rays.y), ref_fin["y"], atol=1e-9)
        np.testing.assert_allclose(be.to_numpy(lens.surfaces.x), ref_rec["x"], atol=1e-9)
    # the only thing handed down a level: the in-kernel launch generation covers paraxial aiming only, so the
    # reference's aimer produced the launch rays (through the wrappers above) and SurfaceGroup.trace carried the trace
    assert set(P.stats()) <= {"fused launch: non-paraxial ray aiming"}, P.stats()


def test_multi_wavelength_and_zernike_error(plugin):
    P, eng, be = plugin
    from optiland.samples.objectives import DoubleGauss

    lens = DoubleGauss()
    n = 30
    Px = np.linspace(-0.5, 0.5, n)
    wl = np.tile([0.4861, 0.5876, 0.6563], n // 3)
    rays = lens.ray_tracer.ray_generator.generate_rays(be.zeros(n), be.zeros(n), be.array(Px), be.zeros(n), be.array(wl))
    lens.surfaces.trace(rays)
    be.set_backend("numpy")
    ref = DoubleGauss()
    r2 = ref.ray_tracer.ray_generator.generate_rays(np.zeros(n), np.zeros(n), Px, np.zeros(n), wl)
    ref.surfaces.trace(r2)
    be.set_backend("torch")
    np.testing.assert_allclose(be.to_numpy(rays.opd), np.array(r2.opd), atol=1e-11)


def test_polarized_trace_with_fresnel_coatings(plugin):
    """Config 5 flavour: Fresnel coatings + unpolarized PolarizedRays through Optic.trace; the
    reference's own update_intensity runs on the P matrices the capability returned."""
    P, eng, be = plugin
    from optiland.rays import PolarizationState
    from optiland.samples.objectives import CookeTriplet

    def make():
        lens = CookeTriplet()
        lens.surfaces.set_fresnel_coatings()
        lens.updater.set_polarization(PolarizationState(is_polarized=False))
        return lens

    def trace(lens):
        return lens.trace(0.0, 0.7, 0.55, 5, "hexapolar")

    be.set_backend("numpy")
    ref = make()
    r_ref = trace(ref)
    ref_i, ref_p = np.array(r_ref.i), np.array(r_ref.p)
    be.set_backend("torch")
    n0 = len(eng.calls)
    lens = make()
    rays = trace(lens)
    assert len(eng.calls) == n0 + 1 and type(rays).__name__ == "PolarizedRays"
    np.testing.assert_allclose(be.to_numpy(rays.i), ref_i, atol=1e-12)
    np.testing.assert_allclose(rays.p.detach().cpu().numpy(), ref_p, atol=1e-12)
    assert float(ref_i.max()) < 0.8  # Fresnel losses really applied


def _c5_lens(state=None):
    """Config 5's system: Zernike freeform singlet + Fresnel coatings + PolarizedRays (oracle/make_golden.py)."""
    from optiland.rays import PolarizationState

    from oracle.make_golden import zernike_singlet

    lens = zernike_singlet("fringe", fresnel=True)
    if state is not None:
        lens.updater.set_polarization(PolarizationState(is_polarized=True, Ex=state[0], Ey=state[1], phase_x=state[2],
                                                        phase_y=state[3]))
    return lens


@pytest.mark.parametrize("state", [None, (1.0, 0.5, 0.0, 0.3)], ids=["unpolarized", "elliptical"])
def test_config5_polarized_call_shapes_go_through_the_fused_launch(plugin, state):
    """Config 5 through the drop-in, zero declines: Optic.trace and trace_generic (per-ray fields and wavelengths) on
    the Zernike + Fresnel system with optic.polarization set produce PolarizedRays from ONE fused launch each --
    records, P matrices and the update_intensity epilogue -- equal to the NumPy reference."""
    P, eng, be = plugin
    rng = np.random.default_rng(11)
    n = 90
    Px, Py = rng.uniform(-0.6, 0.6, n), rng.uniform(-0.6, 0.6, n)
    Hx, Hy = rng.uniform(-0.7, 0.7, n), rng.uniform(-1.0, 1.0, n)
    wl = np.asarray([0.48, 0.55, 0.65])[rng.integers(0, 3, n)]

    def t_single(lens):
        return lens.trace(Hx=0.0, Hy=1.0, wavelength=0.55, num_rays=6, distribution="hexapolar")

    def t_generic(lens):
        a = lambda v: be.array(v)  # noqa: E731
        return lens.trace_generic(a(Hx), a(Hy), a(Px), a(Py), a(wl))

    for trace, n_rays in ((t_single, None), (t_generic, n)):
        be.set_backend("numpy")
        ref = _c5_lens(state)
        r_ref = trace(ref)
        want = {k: np.array(getattr(r_ref, k)) for k in ("x", "y", "z", "L", "M", "N", "i", "opd", "p")}
        want_rec = {k: np.array(getattr(ref.surfaces, k)) for k in ("x", "y", "opd", "intensity")}
        be.set_backend("torch")
        P.stats(reset=True)
        n0 = len(eng.calls)
        lens = _c5_lens(state)
        rays = trace(lens)
        new = eng.calls[n0:]
        assert len(new) == 1 and new[0][0] == "pupil", (new, P.stats())
        assert P.stats() == {} and type(rays).__name__ == "PolarizedRays"
        for k in ("x", "y", "z", "L", "M", "N", "opd"):
            np.testing.assert_allclose(be.to_numpy(getattr(rays, k)), want[k], rtol=0, atol=2e-9, err_msg=k)
        np.testing.assert_allclose(be.to_numpy(rays.i), want["i"], rtol=0, atol=1e-11)
        np.testing.assert_allclose(rays.p.detach().cpu().numpy(), want["p"], rtol=0, atol=1e-10)
        for k, v in want_rec.items():
            np.testing.assert_allclose(be.to_numpy(getattr(lens.surfaces, k)), v, rtol=0, atol=2e-9, err_msg=k)
        if trace is t_single:
            assert float(want["i"].max()) < 0.97          # update_intensity ran: Fresnel losses applied
        else:
            assert float(want["i"].min()) > 0.99          # trace_generic leaves the geometric intensity (no update)
        # the reference's own methods keep working on the returned object
        ef = rays.get_exit_fields(lens.polarization_state)
        be.set_backend("numpy")
        ef_ref = r_ref.get_exit_fields(ref.polarization_state)
        be.set_backend("torch")
        for a, b in zip(ef, ef_ref):
            np.testing.assert_allclose(a.detach().cpu().numpy(), np.array(b), rtol=0, atol=1e-10)


def test_config5_opd_maps_five_fields_three_wavelengths(plugin):
    """Config 5 as BASELINE.json states it: the Wavefront analysis (chief-ray strategy) of the polarized Zernike +
    Fresnel system for 5 fields x 3 wavelengths; every OPD map within 1e-5 waves of the NumPy reference, the exit
    fields and P matrices handed on, every map from one fused wavefront launch and nothing declined."""
    P, eng, be = plugin
    from optiland.wavefront import Wavefront

    fields = [(0.0, 0.0), (0.0, 0.5), (0.0, 1.0), (0.5, 0.5), (-0.7, 0.3)]
    wls = [0.48, 0.55, 0.65]

    def run(lens):
        w = Wavefront(lens, fields=fields, wavelengths=wls, num_rays=10, distribution="hexapolar", strategy="chief_ray")
        out = {}
        for f in fields:
            for wl in wls:
                d = w.get_data(f, wl)
                out[(f, wl)] = {k: np.array(be.to_numpy(getattr(d, k)), dtype=np.float64)
                                for k in ("opd", "pupil_x", "pupil_y", "pupil_z", "intensity")}
                out[(f, wl)]["p"] = np.array(d.prt_matrix.detach().cpu().numpy() if hasattr(d.prt_matrix, "detach") else d.prt_matrix)
                out[(f, wl)]["E"] = [np.array(e.detach().cpu().numpy() if hasattr(e, "detach") else e) for e in d.E_exits]
        return out

    be.set_backend("numpy")
    want = run(_c5_lens())
    be.set_backend("torch")
    P.stats(reset=True)
    n0 = len(eng.calls)
    got = run(_c5_lens())
    assert sum(1 for c in eng.calls[n0:] if c[0] == "wavefront") == 15, eng.calls[n0:]
    assert P.stats() == {}, P.stats()
    worst = 0.0
    for key in want:
        worst = max(worst, float(np.max(np.abs(got[key]["opd"] - want[key]["opd"]))))
        for k in ("pupil_x", "pupil_y", "pupil_z", "intensity"):
            np.testing.assert_allclose(got[key][k], want[key][k], rtol=0, atol=1e-9, err_msg=str((key, k)))
        np.testing.assert_allclose(got[key]["p"], want[key]["p"], rtol=0, atol=1e-10)
        for a, b in zip(got[key]["E"], want[key]["E"]):
            np.testing.assert_allclose(a, b, rtol=0, atol=1e-10)
    assert worst <= 1e-5, worst          # waves: BASELINE.json config 5's tolerance


def test_autograd_through_the_capability_matches_reference_eager_graph(plugin):
    """Config 3 through the drop-in: with be.grad_mode on, d(RMS spot)/d(radius, conic, thickness-z) obtained
    via Optic.trace -> capability (one custom autograd Function) equals the reference's own eager autograd,
    INCLUDING the dependence of the launch rays on the radii through paraxial ray aiming."""
    import torch

    P, eng, be = plugin
    from oracle.make_golden import reverse_telephoto_asphere

    def run(lens):
        rays = lens.trace(0.0, 0.7, 0.5876, 6, "hexapolar")
        x = lens.surfaces.x[-1, :]
        y = lens.surfaces.y[-1, :]
        loss = torch.sqrt(torch.mean((x - torch.mean(x)) ** 2 + (y - torch.mean(y)) ** 2))
        loss.backward()
        out = {"loss": float(loss.detach())}
        for s in (1, 2, 13):
            g = lens.surfaces.surfaces[s].geometry
            out[f"r{s}"] = float(g.radius.grad)
        out["k13"] = float(lens.surfaces.surfaces[13].geometry.k.grad)
        out["z1"] = float(lens.surfaces.surfaces[1].geometry.cs.z.grad)
        return out

    be.grad_mode.enable()
    try:
        n0 = len(eng.calls)
        got = run(reverse_telephoto_asphere(1e-12))
        assert any(c[0] == "grad" for c in eng.calls[n0:])
        P.uninstall()                       # the reference's own eager graph
        ref = run(reverse_telephoto_asphere(1e-12))
    finally:
        be.grad_mode.disable()
    assert got["loss"] == pytest.approx(ref["loss"], rel=1e-9)
    for k in ref:
        assert got[k] == pytest.approx(ref[k], rel=2e-6), k


def test_autograd_tilt_and_decenter_variables_match_reference_eager_graph(plugin):
    """Tilted / decentered surfaces with be.grad_mode on: d(RMS spot)/d(rx, ry, rz, dx, dy, radius) through the
    capability (adjoint kernel's dLoss/dR chained to the live angle tensors) equals the reference's own eager
    autograd -- including its quirk that an angle that is exactly 0 gets no gradient."""
    import torch

    P, eng, be = plugin
    from optiland import optic as _optic

    def make():
        lens = _optic.Optic()
        lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
        lens.surfaces.add(index=1, radius=50.0, thickness=5.0, material="N-BK7", is_stop=True,
                          dx=0.3, dy=-0.2, rx=0.02, ry=-0.015)
        lens.surfaces.add(index=2, radius=-80.0, thickness=30.0, rz=0.4, rx=-0.01, conic=-0.8)
        lens.surfaces.add(index=3, radius=be.inf, thickness=-25.0, material="mirror", rx=np.pi / 4)
        lens.surfaces.add(index=4, radius=be.inf, thickness=0.0, rx=np.pi / 2, dy=0.5)
        lens.set_aperture(aperture_type="EPD", value=10.0)
        lens.fields.set_type(field_type="angle")
        lens.fields.add(y=0)
        lens.fields.add(y=3)
        lens.wavelengths.add(value=0.6, is_primary=True)
        return lens

    def run(lens):
        lens.trace(0.0, 1.0, 0.6, 5, "hexapolar")
        x = lens.surfaces.x[-1, :]
        y = lens.surfaces.y[-1, :]
        z = lens.surfaces.z[-1, :]
        loss = torch.sqrt(torch.mean((x - torch.mean(x)) ** 2 + (y - torch.mean(y)) ** 2 + (z - torch.mean(z)) ** 2))
        loss.backward()
        out = {"loss": float(loss.detach())}
        for s in (1, 2, 3):
            cs = lens.surfaces.surfaces[s].geometry.cs
            for k in ("rx", "ry", "rz", "x", "y"):
                g = getattr(cs, k).grad
                out[f"{k}{s}"] = 0.0 if g is None else float(g)
        out["r1"] = float(lens.surfaces.surfaces[1].geometry.radius.grad)
        return out

    be.grad_mode.enable()
    try:
        n0 = len(eng.calls)
        got = run(make())
        assert any(c[0] == "grad" for c in eng.calls[n0:]), P.stats()
        P.uninstall()
        ref = run(make())
    finally:
        be.grad_mode.disable()
    assert got["loss"] == pytest.approx(ref["loss"], rel=1e-9)
    scale = max(abs(v) for k, v in ref.items() if k != "loss")
    for k in ref:
        assert got[k] == pytest.approx(ref[k], rel=2e-6, abs=1e-9 * scale), (k, got[k], ref[k])
    assert ref["rx1"] != 0 and ref["rz2"] != 0 and ref["rx3"] != 0      # the tilt gradients are really there
    assert ref["rz1"] == 0 and got["rz1"] == 0                           # zero angle: skipped by the reference


def test_autograd_zernike_and_polynomial_coefficient_variables(plugin):
    """Freeform optimisation variables through the capability: d(RMS spot)/d(Zernike coefficient), d/d(polynomial
    coefficient), d/d(Chebyshev coefficient), d/d(radius, conic) of the freeform surface -- forward kernel + the polynomial-family adjoint
    (olb_trace_bwd_* grad_tables: table gradients mapped back to the live coefficient tensors) -- equal the reference's own
    eager autograd, with the coefficients set the way ZernikeCoeffVariable / PolynomialCoeffVariable set them
    (optimization/variable/zernike_coeff.py:71-95: ``geometry.coefficients[i] = value``; polynomial_coeff.py:77-81 and its
    subclass chebyshev_coeff.py: ``geometry.coefficients[i][j] = value``)."""
    import torch

    P, eng, be = plugin
    from optiland import optic as _optic

    from oracle.make_golden import zernike_singlet

    def make_poly():
        lens = _optic.Optic()
        lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
        lens.surfaces.add(index=1, radius=35.0, thickness=5.0, material="N-BK7", is_stop=True, surface_type="polynomial",
                          conic=-0.3, coefficients=[[0.0, 1e-3, -2e-4], [2e-3, -3e-4, 1e-5], [4e-4, 2e-5, -1e-6]], tol=1e-12)
        lens.surfaces.add(index=2, radius=-70.0, thickness=40.0)
        lens.surfaces.add(index=3)
        lens.set_aperture(aperture_type="EPD", value=12.0)
        lens.fields.set_type(field_type="angle")
        lens.fields.add(y=0)
        lens.fields.add(y=4)
        lens.wavelengths.add(value=0.55, is_primary=True)
        return lens

    def make_cheb():
        lens = _optic.Optic()
        lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
        lens.surfaces.add(index=1, radius=40.0, thickness=5.0, material="N-BK7", is_stop=True, surface_type="chebyshev",
                          conic=-0.2, coefficients=[[0.0, 2e-3, -5e-4], [1e-3, -4e-4, 1e-4], [3e-4, 1e-4, -5e-5]],
                          norm_x=9.0, norm_y=11.0, tol=1e-12)
        lens.surfaces.add(index=2, radius=-70.0, thickness=40.0)
        lens.surfaces.add(index=3)
        lens.set_aperture(aperture_type="EPD", value=12.0)
        lens.fields.set_type(field_type="angle")
        lens.fields.add(y=0)
        lens.fields.add(y=4)
        lens.wavelengths.add(value=0.55, is_primary=True)
        return lens

    def run(make, kind):
        lens = make()
        g = lens.surfaces.surfaces[1].geometry
        leaves = {}
        if kind == "zernike":
            for idx in (3, 8, 12):
                leaf = torch.tensor(float(g.coefficients[idx]), dtype=torch.float64, device=g.coefficients.device, requires_grad=True)
                g.coefficients[idx] = leaf
                leaves[f"c{idx}"] = leaf
        else:
            for (i, j) in ((0, 1), (1, 1), (2, 0)):
                leaf = torch.tensor(float(g.coefficients[i][j]), dtype=torch.float64, device=g.coefficients.device, requires_grad=True)
                g.coefficients[i][j] = leaf
                leaves[f"c{i}{j}"] = leaf
        lens.trace(0.0, 1.0, 0.55, 7, "hexapolar")
        x = lens.surfaces.x[-1, :]
        y = lens.surfaces.y[-1, :]
        loss = torch.sqrt(torch.mean((x - torch.mean(x)) ** 2 + (y - torch.mean(y)) ** 2))
        loss.backward()
        out = {"loss": float(loss.detach())}
        out.update({k: float(v.grad) for k, v in leaves.items()})
        out["radius"] = float(g.radius.grad)
        out["conic"] = float(g.k.grad)
        return out

    def fd_reference(make, kind, which, h):
        """Central difference of the loss computed by the reference's NumPy backend (launch rays re-aimed, as in run())."""
        vals = []
        for sign in (+1, -1):
            be.set_backend("numpy")
            lens = make()
            g = lens.surfaces.surfaces[1].geometry
            if which == "radius":
                g.radius = g.radius + sign * h
            elif which == "conic":
                g.k = g.k + sign * h
            elif kind == "zernike":
                g.coefficients[int(which[1:])] += sign * h
            else:
                g.coefficients[int(which[1])][int(which[2])] += sign * h
            lens.trace(0.0, 1.0, 0.55, 7, "hexapolar")
            x, y = np.array(lens.surfaces.x[-1, :]), np.array(lens.surfaces.y[-1, :])
            vals.append(float(np.sqrt(np.mean((x - x.mean()) ** 2 + (y - y.mean()) ** 2))))
            be.set_backend("torch")
        return (vals[0] - vals[1]) / (2 * h)

    be.grad_mode.enable()
    try:
        for make, kind in ((lambda: zernike_singlet("fringe"), "zernike"), (make_poly, "polynomial"),
                           (make_cheb, "chebyshev")):
            P.install(engine=eng)
            P.stats(reset=True)
            n0 = len(eng.calls)
            got = run(make, kind)
            assert any(c[0] == "grad" for c in eng.calls[n0:]), (kind, P.stats())
            P.uninstall()
            try:
                ref = run(make, kind)
            except RuntimeError as e:
                # the STOCK reference cannot differentiate a Zernike surface at all: its radial terms use `//` on
                # tensors ("derivative for aten::floor_divide is not implemented") -- compare with central differences
                # of its NumPy forward pass instead
                assert kind == "zernike" and "floor_divide" in str(e)
                be.grad_mode.disable()
                ref = {k: fd_reference(make, kind, k, 1e-6 if k != "radius" else 1e-4) for k in got if k != "loss"}
                ref["loss"] = got["loss"]
                be.grad_mode.enable()
                tol = 2e-4
            else:
                tol = 5e-6
            assert got["loss"] == pytest.approx(ref["loss"], rel=1e-9)
            scale = max(abs(v) for k, v in ref.items() if k != "loss")
            for k in ref:
                assert got[k] == pytest.approx(ref[k], rel=tol, abs=tol * 1e-2 * scale), (kind, k, got[k], ref[k])
    finally:
        be.grad_mode.disable()


def test_autograd_trace_generic_with_several_wavelengths_in_one_call(plugin):
    """``trace_generic`` with a per-ray wavelength array while gradients are wanted: the batch is split by wavelength
    (one forward + one adjoint launch each, with that wavelength's live indices) and the records come back in the
    caller's ray order.  Loss = RMS spot over all rays; gradients w.r.t. a radius, a thickness (surface z), a conic, the
    Abbe material's index AND Abbe number (n(lambda) differs per wavelength and is a differentiable function of both:
    materials/abbe.py:45-76, the polynomial model's leaves) equal the reference's own eager autograd."""
    import torch

    P, eng, be = plugin
    from optiland import optic as _optic
    from optiland.materials import AbbeMaterial

    def make():
        lens = _optic.Optic()
        lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
        lens.surfaces.add(index=1, radius=45.0, thickness=6.0, material=AbbeMaterial(1.62, 45.0, model="polynomial"), is_stop=True, conic=-0.4)
        lens.surfaces.add(index=2, radius=-60.0, thickness=3.0, material="SF5")
        lens.surfaces.add(index=3, radius=-150.0, thickness=60.0)
        lens.surfaces.add(index=4)
        lens.set_aperture(aperture_type="EPD", value=14.0)
        lens.fields.set_type(field_type="angle")
        lens.fields.add(y=0)
        lens.fields.add(y=5)
        for wv, prim in ((0.4861, False), (0.5876, True), (0.6563, False)):
            lens.wavelengths.add(value=wv, is_primary=prim)
        return lens

    rng = np.random.default_rng(3)
    n = 60
    r, th = np.sqrt(rng.uniform(size=n)), rng.uniform(0, 2 * np.pi, size=n)
    Px, Py = r * np.cos(th), r * np.sin(th)
    Hy = rng.choice([0.0, 0.7, 1.0], size=n)
    wv = rng.choice([0.4861, 0.5876, 0.6563], size=n)        # interleaved: the regrouping has to undo a real permutation

    def run(lens):
        dev = lens.surfaces.surfaces[1].geometry.radius.device
        t = lambda a: torch.as_tensor(a, dtype=torch.float64, device=dev)  # noqa: E731
        cs2 = lens.surfaces.surfaces[2].geometry.cs
        cs2.z = torch.tensor(float(cs2.z), dtype=torch.float64, device=dev, requires_grad=True)   # a leaf, like a thickness variable
        rays = lens.trace_generic(t(np.zeros(n)), t(Hy), t(Px), t(Py), t(wv))
        x, y = lens.surfaces.x[-1, :], lens.surfaces.y[-1, :]
        loss = torch.sqrt(torch.mean((x - torch.mean(x)) ** 2 + (y - torch.mean(y)) ** 2)) + 1e-3 * torch.mean(lens.surfaces.opd[-1, :])
        loss.backward()
        g1, mat = lens.surfaces.surfaces[1].geometry, lens.surfaces.surfaces[1].material_post
        out = {"loss": float(loss.detach()), "radius1": float(g1.radius.grad), "conic1": float(g1.k.grad),
               "z2": float(lens.surfaces.surfaces[2].geometry.cs.z.grad), "index": float(mat.model.index.grad),
               "abbe": float(mat.model.abbe.grad)}
        return out, be.to_numpy(rays.x), be.to_numpy(lens.surfaces.y)

    be.grad_mode.enable()
    try:
        P.stats(reset=True)
        n0 = len(eng.calls)
        got, gx, gy = run(make())
        grads = [c for c in eng.calls[n0:] if c[0] == "grad"]
        assert len(grads) == 3 and sum(c[2] for c in grads) == n, (grads, P.stats())
        assert not P.stats(), P.stats()
        P.uninstall()                       # the reference's own eager graph
        ref, rx, ry = run(make())
    finally:
        be.grad_mode.disable()
    assert np.allclose(gx, rx, rtol=0, atol=1e-10) and np.allclose(gy, ry, rtol=0, atol=1e-10, equal_nan=True)
    assert got["loss"] == pytest.approx(ref["loss"], rel=1e-10)
    for k in ref:
        assert got[k] == pytest.approx(ref[k], rel=5e-6), (k, got[k], ref[k])


def test_surface_group_trace_capability_when_launch_fusion_is_off(plugin):
    """With the RealRayTracer.trace wrapper disabled the SurfaceGroup.trace wrapper carries the call
    (launch rays from the reference's own RayGenerator)."""
    P, eng, be = plugin
    from optiland.samples.objectives import DoubleGauss

    P._state["fuse_launch"] = False
    try:
        lens = DoubleGauss()
        rays = lens.trace(Hx=0.0, Hy=0.7, wavelength=0.5876, num_rays=5, distribution="hexapolar")
        assert eng.calls[-1][0] == 13
    finally:
        P._state["fuse_launch"] = True
    n0 = len(eng.calls)
    lens2 = DoubleGauss()
    rays2 = lens2.trace(Hx=0.0, Hy=0.7, wavelength=0.5876, num_rays=5, distribution="hexapolar")
    assert eng.calls[n0][0] == "pupil"
    np.testing.assert_allclose(be.to_numpy(rays2.y), be.to_numpy(rays.y), atol=1e-11)
    np.testing.assert_allclose(be.to_numpy(lens2.surfaces.opd), be.to_numpy(lens.surfaces.opd), atol=1e-11)


def test_huygens_psf_strategy_is_routed_through_the_engine(plugin):
    """f-3: HuygensPSF on the torch backend calls the capability instead of TorchSummation's eager loop;
    same Strehl-normalised PSF as the reference's NumPy/Numba path."""
    P, eng, be = plugin
    from optiland.psf import HuygensPSF
    from optiland.samples.objectives import CookeTriplet

    be.set_backend("numpy")
    ref = np.array(HuygensPSF(CookeTriplet(), field=(0, 0.7), wavelength=0.55, num_rays=24, image_size=16).psf)
    be.set_backend("torch")
    n0 = len(eng.calls)
    got = HuygensPSF(CookeTriplet(), field=(0, 0.7), wavelength=0.55, num_rays=24, image_size=16).psf
    assert any(c[0] == "psf" for c in eng.calls[n0:])
    np.testing.assert_allclose(be.to_numpy(got), ref, rtol=0, atol=1e-8 * ref.max())


def test_fft_psf_takes_its_pupil_function_from_the_fused_wavefront_epilogue(plugin):
    """FFTPSF (psf/fft.py:123-227): its wavefront data comes from ``Wavefront.get_data`` -- under the plugin ONE fused
    launch (launch generation + trace + OPD against the reference sphere + intensity) -- and the gridding passes on
    either side of the library FFT are one kernel each: ``olb_fft_pupil_*`` writes the zero-padded pupil function
    A exp(-2 pi i OPD) (masked scatter + reshape + pad), ``olb_fft_psf_accumulate_*`` reads the spectrum once (|.|^2,
    fftshift, sum over wavelengths, normalisation).  Same PSF as the NumPy reference; ``self.pupils`` keeps its
    meaning (num_rays x num_rays complex arrays) and equals the reference's."""
    P, eng, be = plugin
    from optiland.psf import FFTPSF
    from optiland.samples.objectives import CookeTriplet

    for kw in (dict(field=(0, 0.7), wavelength=0.55, num_rays=64, grid_size=128),
               dict(field=(0, 1.0), wavelength=0.48, num_rays=33, grid_size=77)):       # odd sizes (pad 22 / 22, shift 38)
        be.set_backend("numpy")
        r = FFTPSF(CookeTriplet(), **kw)
        ref, ref_pupils = np.array(r.psf), [np.array(p) for p in r.pupils]
        be.set_backend("torch")
        n0 = len(eng.calls)
        P.stats(reset=True)
        psf = FFTPSF(CookeTriplet(), **kw)
        kinds = [c[0] for c in eng.calls[n0:]]
        assert "wavefront" in kinds and kinds.count("fft_pupil") == len(ref_pupils) == kinds.count("fft_psf"), kinds
        np.testing.assert_allclose(be.to_numpy(psf.psf), ref, rtol=0, atol=2e-6 * ref.max())
        assert len(psf.pupils) == len(ref_pupils)
        for got_p, ref_p in zip(psf.pupils, ref_pupils):
            assert tuple(got_p.shape) == ref_p.shape
            np.testing.assert_allclose(be.to_numpy(got_p), ref_p, rtol=0, atol=1e-6)
        assert float(psf._get_normalization()) == float(np.sum(np.abs(ref_pupils[0]) > 0) ** 2)
        # a caller that REPLACES the pupils gets the reference's own code on them (no stale padded buffers)
        psf.pupils = [p * 0.5 for p in psf.pupils]
        n1 = len(eng.calls)
        np.testing.assert_allclose(be.to_numpy(psf._compute_psf()), 0.25 * ref, rtol=0, atol=2e-6 * ref.max())
        assert not [c for c in eng.calls[n1:] if c[0] == "fft_psf"]
    # gradients wanted: the reference's eager ops
    be.grad_mode.enable()
    try:
        n2 = len(eng.calls)
        FFTPSF(CookeTriplet(), field=(0, 0.0), wavelength=0.55, num_rays=32, grid_size=64)
        assert not [c for c in eng.calls[n2:] if c[0] in ("fft_pupil", "fft_psf")]
    finally:
        be.grad_mode.disable()


def test_launch_form_reproduces_the_reference_ray_generator_known_answers():
    """the reference's tests/test_rays.py:685-714: TessarLens, H = (0.5, 0.5), P = (0.1, 0.1), (0.2, 0.2) -- the
    reference's hard-coded launch rays, reproduced by pack.launch_scalars + launch.pupil_affine (the form the kernel
    evaluates)."""
    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be
    from optiland.samples.objectives import TessarLens

    from optiland_b200.launch import launch_from_affine, pupil_affine
    from optiland_b200.pack import launch_scalars

    be.set_backend("numpy")
    sc = launch_scalars(TessarLens(), 0.5, 0.5)
    x, y, z, L, M, N = launch_from_affine(np.array([0.1, 0.2]), np.array([0.1, 0.2]), pupil_affine(sc))
    np.testing.assert_allclose(x, [-0.23535066, -0.1909309], atol=1e-8)
    np.testing.assert_allclose(y, [-0.23535066, -0.1909309], atol=1e-8)
    np.testing.assert_allclose(z, [-0.88839505, -0.88839505], atol=1e-8)
    np.testing.assert_allclose(L, [0.17519154, 0.17519154], atol=1e-8)
    np.testing.assert_allclose(M, [0.17519154, 0.17519154], atol=1e-8)
    np.testing.assert_allclose(N, [0.96882189, 0.96882189], atol=1e-8)
