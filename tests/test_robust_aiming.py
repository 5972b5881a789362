"""Robust ray aiming (Optiland's ``RobustRayAimer``, mode ``"robust"``) with every solve of its continuation as ONE launch of
the aim kernel (include/olb.h ``OlbAimCall``, csrc/olb_aim.cuh).

CPU part: the host instantiation of the solve (tests/hostcheck/hostcheck_aim.cpp) against the reference's own
``IterativeRayAimer.aim_rays`` on live systems, forced failures, and the plugin's restated robust aimer end to end through
a test engine on that instantiation (``oracle/aim_engines.py``).  GPU part (``gpu`` marker): the CUDA solve against the
host instantiation for each kernel variant, and ``[cuda]`` robust traces against NumPy."""
import numpy as np
import pytest

from oracle.ref_import import reference_available

pytestmark = pytest.mark.skipif(not reference_available(), reason="reference not present on this box")

ROBUST = ("ProjectionLens120FOV", "ProjectionLens160FOV", "WideAngle170FOV")
KEYS = ("x", "y", "z", "L", "M", "N")


@pytest.fixture
def torch_backend():
    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be

    from optiland_b200 import plugin as P

    P.uninstall()
    be.set_backend("torch")
    be.set_device("cpu")
    be.set_precision("float64")
    be.grad_mode.disable()
    yield be
    P.uninstall()
    be.set_backend("numpy")


def _sample(name):
    from optiland.samples import objectives

    return getattr(objectives, name)()


def _hexapolar(rings=4):
    px, py = [0.0], [0.0]
    for r in range(1, rings + 1):
        for k in range(6 * r):
            a = 2 * np.pi * k / (6 * r)
            px.append(r / rings * np.cos(a))
            py.append(r / rings * np.sin(a))
    return np.array(px), np.array(py)


def _finite_object(be):
    from optiland import optic

    lens = optic.Optic()
    lens.surfaces.add(index=0, thickness=80.0)
    lens.surfaces.add(index=1, radius=40.0, thickness=6.0, material="N-BK7")
    lens.surfaces.add(index=2, radius=-40.0, thickness=4.0)
    lens.surfaces.add(index=3, thickness=50.0, is_stop=True)
    lens.surfaces.add(index=4)
    lens.set_aperture(aperture_type="objectNA", value=0.08)
    lens.fields.set_type(field_type="object_height")
    lens.fields.add(y=0.0)
    lens.fields.add(y=6.0)
    lens.wavelengths.add(value=0.55, is_primary=True)
    return lens


def _tilted_stop(be):
    from optiland import optic

    lens = optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=45.0, thickness=6.0, material="N-BK7")
    lens.surfaces.add(index=2, radius=-70.0, thickness=5.0)
    lens.surfaces.add(index=3, thickness=45.0, is_stop=True, dy=0.4, dx=-0.2, rx=0.03, ry=-0.02)
    lens.surfaces.add(index=4)
    lens.set_aperture(aperture_type="EPD", value=12.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=8.0)
    for w, p in ((0.48, False), (0.55, True), (0.65, False)):
        lens.wavelengths.add(value=w, is_primary=p)
    return lens


def _doe_before_stop(be):
    from optiland import optic
    from optiland.phase import RadialPhaseProfile

    lens = optic.Optic()
    lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
    lens.surfaces.add(index=1, radius=45.0, thickness=6.0, material="N-BK7",
                      phase_profile=RadialPhaseProfile([-1.0, 2e-4]))
    lens.surfaces.add(index=2, radius=-70.0, thickness=5.0)
    lens.surfaces.add(index=3, thickness=45.0, is_stop=True)
    lens.surfaces.add(index=4)
    lens.set_aperture(aperture_type="EPD", value=12.0)
    lens.fields.set_type(field_type="angle")
    lens.fields.add(y=0.0)
    lens.fields.add(y=6.0)
    lens.wavelengths.add(value=0.55, is_primary=True)
    return lens


def _zernike_stop(be, norm_radius):
    from oracle.make_golden import zernike_singlet

    return zernike_singlet("fringe", norm_radius=norm_radius)


def _aim_inputs(lens, hx, hy, t, wl=None, max_iter=None):
    """Everything one solve needs: the reference's aimer, its targets and paraxial guess, and the host solve's table
    and scalars (computed as the plugin computes them)."""
    import optiland.backend as be
    from optiland.rays.ray_aiming.initialization import get_stop_radius_strategy
    from optiland.rays.ray_aiming.iterative import IterativeRayAimer

    from optiland_b200 import table as T
    from optiland_b200.pack import pack_surface_group

    it = IterativeRayAimer(lens)
    if max_iter is not None:
        it.max_iter = max_iter
    px, py = _hexapolar()
    n = px.size
    Px, Py = be.array(px * t), be.array(py * t)
    H = (be.array(np.full(n, hx * t)), be.array(np.full(n, hy * t)))
    if wl is None:
        wl = lens.primary_wavelength
    guess = it._paraxial_aimer.aim_rays(H, wl, (Px, Py))
    stop = lens.surfaces.stop_index
    inf = bool(getattr(lens.object_surface, "is_infinite", False))
    start = 1 if inf else 0
    wls = np.unique(np.atleast_1d(be.to_numpy(be.as_array_1d(wl))))
    full = pack_surface_group(lens.surfaces, wls)
    table = T.SurfaceTable(full.surfaces[start:stop + 1], full.wavelengths)
    r_stop = float(get_stop_radius_strategy(lens, "iterative").calculate_stop_radius())
    wl_mean = be.mean(wl) if hasattr(wl, "__len__") else wl
    J = it._get_paraxial_jacobian(float(wl_mean), stop, inf)
    J = 1e-12 if abs(J) < 1e-12 else float(J)
    return dict(it=it, H=H, Px=Px, Py=Py, wl=wl, guess=guess, table=table, r_stop=r_stop, J=J, inf=inf)


def _host_solve(a, guess=None, dtype=np.float64):
    import optiland.backend as be

    from oracle.hostcheck_aim import run_aim

    g = {k: be.to_numpy(be.as_array_1d(v)) for k, v in zip(KEYS, guess if guess is not None else a["guess"])}
    g["w"] = np.broadcast_to(be.to_numpy(be.as_array_1d(a["wl"])), g["x"].shape)
    return run_aim(a["table"], g, be.to_numpy(a["Px"]), be.to_numpy(a["Py"]), 0, a["table"].num_surfaces, a["r_stop"],
                   a["J"], a["it"].tol, a["it"].max_iter, a["inf"], dtype=dtype)


def _reference_solve(a, guess=None):
    import optiland.backend as be

    try:
        out = a["it"].aim_rays(a["H"], a["wl"], (a["Px"], a["Py"]),
                               initial_guess=guess if guess is not None else a["guess"])
    except ValueError:
        return None
    return {k: be.to_numpy(v) for k, v in zip(KEYS, out)}


def _assert_same(ref, sol, status, scale, what):
    assert (ref is None) == (status != 0), (what, status)
    if ref is None:
        return
    for k in KEYS:
        err = float(np.max(np.abs(sol[k] - ref[k])))
        assert err <= 1e-10 * scale, (what, k, err)


def _scale(lens):
    import optiland.backend as be

    z = be.to_numpy(lens.surfaces.positions).ravel()
    return max(1.0, float(np.max(np.abs(z[np.isfinite(z)]))))


# ---- host solve == IterativeRayAimer.aim_rays ------------------------------------------------------------------------

@pytest.mark.parametrize("t", [0.25, 0.6, 1.0])
@pytest.mark.parametrize("name", ROBUST)
def test_host_solve_equals_iterative_aimer_on_robust_samples(torch_backend, name, t):
    lens = _sample(name)
    outcomes = []
    for f in lens.fields.get_field_coords():
        a = _aim_inputs(lens, float(f[0]), float(f[1]), t)
        sol, status, _ = _host_solve(a)
        ref = _reference_solve(a)
        _assert_same(ref, sol, status, _scale(lens), (name, tuple(f), t))
        outcomes.append(ref is not None)
    if t == 0.25:
        assert all(outcomes)      # small steps of the continuation converge: the solutions are compared


@pytest.mark.parametrize("build,variant", [
    (_finite_object, "closed form"), (_tilted_stop, "closed form"), (_doe_before_stop, "superset"),
    (lambda be: _zernike_stop(be, 12.0), "general")])
def test_host_solve_equals_iterative_aimer_on_live_systems(torch_backend, build, variant):
    be = torch_backend
    lens = build(be)
    converged = 0
    for f in lens.fields.get_field_coords():
        for t in (0.5, 1.0):
            a = _aim_inputs(lens, float(f[0]), float(f[1]), t)
            sol, status, v = _host_solve(a)
            assert v == variant
            ref = _reference_solve(a)
            _assert_same(ref, sol, status, _scale(lens), (variant, tuple(f), t))
            converged += ref is not None
            assert not a["inf"] or np.array_equal(sol["L"], be.to_numpy(a["guess"][3]))   # infinite: only (x, y) move
    assert converged >= 2


def test_host_solve_multi_wavelength(torch_backend):
    be = torch_backend
    lens = _tilted_stop(be)
    n = _hexapolar()[0].size
    wl = be.array(np.array([0.48, 0.55, 0.65])[np.arange(n) % 3])
    a = _aim_inputs(lens, 0.0, 8.0, 1.0, wl=wl)
    assert a["table"].n_wl == 3
    sol, status, _ = _host_solve(a)
    _assert_same(_reference_solve(a), sol, status, _scale(lens), "trace_generic wavelengths")


def test_finite_object_moves_L_M_and_keeps_N(torch_backend):
    be = torch_backend
    a = _aim_inputs(_finite_object(be), 0.0, 6.0, 1.0)
    sol, status, _ = _host_solve(a)
    assert status == 0 and not a["inf"]
    g = {k: be.to_numpy(v) for k, v in zip(KEYS, a["guess"])}
    for k in ("x", "y", "z", "N"):
        assert np.array_equal(sol[k], g[k]), k
    assert np.max(np.abs(sol["M"] - g["M"])) > 0


# ---- forced failures: the same outcome as the reference's ValueError -------------------------------------------------

def test_nan_start_is_a_failed_solve(torch_backend):
    from optiland_b200 import table as T

    be = torch_backend
    a = _aim_inputs(_tilted_stop(be), 0.0, 8.0, 1.0)
    x = be.to_numpy(a["guess"][0]).copy()
    x[3] = np.nan
    guess = (be.array(x),) + tuple(a["guess"][1:])
    assert _reference_solve(a, guess) is None
    _, status, _ = _host_solve(a, guess)
    assert status == T.ST_AIM_NAN_START


def test_max_iter_one_is_unconverged(torch_backend):
    from optiland_b200 import table as T

    be = torch_backend
    a = _aim_inputs(_sample("WideAngle170FOV"), 0.0, 0.5, 0.5, max_iter=1)
    assert _reference_solve(a) is None
    _, status, _ = _host_solve(a)
    assert status == T.ST_AIM_UNCONVERGED


def test_zernike_range_error_is_a_failed_solve(torch_backend):
    from optiland_b200 import table as T

    be = torch_backend
    a = _aim_inputs(_zernike_stop(be, 5.0), 0.0, 5.0, 1.0)
    assert _reference_solve(a) is None
    _, status, v = _host_solve(a)
    assert v == "general" and status & T.ST_ZERNIKE_RANGE


# ---- the plugin's robust aimer through the host instantiation --------------------------------------------------------

@pytest.fixture
def aim_plugin(torch_backend):
    from oracle.aim_engines import AimDeviceMathEngine
    from optiland_b200 import plugin as P

    eng = AimDeviceMathEngine()
    P.install(engine=eng)
    P.stats(reset=True)
    yield P, eng, torch_backend


class _Spy:
    """Counts the reference's solves (IterativeRayAimer.aim_rays) and subset traces (_trace_subset)."""

    def __init__(self, monkeypatch):
        from optiland.rays.ray_aiming.iterative import IterativeRayAimer

        self.solves = self.subsets = 0
        aim, sub = IterativeRayAimer.aim_rays, IterativeRayAimer._trace_subset

        def aim2(it, *a, **k):
            self.solves += 1
            return aim(it, *a, **k)

        def sub2(it, *a, **k):
            self.subsets += 1
            return sub(it, *a, **k)

        monkeypatch.setattr(IterativeRayAimer, "aim_rays", aim2)
        monkeypatch.setattr(IterativeRayAimer, "_trace_subset", sub2)


def _numpy_records(name, fields):
    import optiland.backend as be

    be.set_backend("numpy")
    ref = _sample(name)
    out = []
    for hx, hy in fields:
        ref.trace(hx, hy, ref.primary_wavelength, 4, "hexapolar")
        out.append({k: np.array(getattr(ref.surfaces, k)) for k in ("x", "y", "z", "L", "M", "N", "opd", "intensity")})
    be.set_backend("torch")
    return out


def _check_records(be, lens, want, what):
    scale = max(1.0, float(np.nanmax(np.abs(np.where(np.isfinite(want["z"]), want["z"], 0.0)))))
    for k, v in want.items():
        g = be.to_numpy(getattr(lens.surfaces, k))
        assert np.array_equal(np.isnan(g), np.isnan(v)), (what, k)
        m = np.isfinite(v)
        assert not m.any() or float(np.max(np.abs(g[m] - v[m]))) <= 1e-10 * scale, (what, k)


@pytest.mark.parametrize("name", ROBUST)
def test_robust_trace_through_device_aim_equals_numpy(aim_plugin, monkeypatch, name):
    P, eng, be = aim_plugin
    lens0 = _sample(name)
    fields = [tuple(float(v) for v in f) for f in lens0.fields.get_field_coords()]
    want = _numpy_records(name, fields)
    spy = _Spy(monkeypatch)
    lens = _sample(name)
    for (hx, hy), w in zip(fields, want):
        # one solve of the reference per aim launch: the reference's body first, counted, then the device path
        P._state["device_aim"] = False
        s0 = spy.solves
        lens.trace(hx, hy, lens.primary_wavelength, 4, "hexapolar")
        ref_solves = spy.solves - s0
        P._state["device_aim"] = True
        spy.subsets = 0
        s0, n0 = spy.solves, len(eng.calls)
        lens.trace(hx, hy, lens.primary_wavelength, 4, "hexapolar")
        aims = sum(1 for c in eng.calls[n0:] if c[0] == "aim")
        assert spy.subsets == 0 and spy.solves == s0, (name, hx, hy)
        assert aims == ref_solves, (name, hx, hy, aims, ref_solves)
        _check_records(be, lens, w, (name, hx, hy))
    assert set(P.stats()) <= {"fused launch: non-paraxial ray aiming"}, P.stats()


def test_widest_field_engine_calls(aim_plugin):
    """WideAngle170FOV at full field: 3935 engine calls per Optic.trace through the reference's body, ~261 here (one aim
    launch per solve, the stop-radius trace once, the final trace)."""
    P, eng, be = aim_plugin
    lens = _sample("WideAngle170FOV")
    n0 = len(eng.calls)
    lens.trace(0.0, 1.0, lens.primary_wavelength, 4, "hexapolar")
    calls = eng.calls[n0:]
    aims = sum(1 for c in calls if c[0] == "aim")
    assert aims > 200 and len(calls) <= aims + 20, (aims, len(calls))


def test_cached_aimer_returns_cached_results_and_reuses_guesses(aim_plugin, monkeypatch):
    """``CachedRayAimer`` around the robust aimer (``set_aiming("robust", cache=True)``): a repeated call returns the
    cached result without a solve; after a change of the system the cached result is the initial guess of one solve.
    The device path makes the reference body's solves, with equal results."""
    from optiland.rays.ray_aiming.cached import CachedRayAimer
    from optiland.rays.ray_aiming.robust import RobustRayAimer

    P, eng, be = aim_plugin
    spy = _Spy(monkeypatch)
    px, py = _hexapolar()
    n = px.size
    args = ((be.array(np.zeros(n)), be.array(np.full(n, 0.7))), 0.5876, (be.array(px), be.array(py)))
    counts, results = {}, {}
    for device in (False, True):
        P._state["device_aim"] = device
        lens = _sample("ProjectionLens120FOV")
        aimer = CachedRayAimer(lens, RobustRayAimer(lens))
        per_call, outs = [], []
        for step in range(3):
            if step == 2:
                lens.surfaces[1].geometry.cs.z = lens.surfaces[1].geometry.cs.z + 1e-4
            s0, n0 = spy.solves, len(eng.calls)
            outs.append(aimer.aim_rays(*args))
            per_call.append(sum(1 for c in eng.calls[n0:] if c[0] == "aim") if device else spy.solves - s0)
        assert outs[1] is outs[0]                                   # the cached tuple itself
        counts[device], results[device] = per_call, outs
    assert counts[True] == counts[False] and counts[True][1] == 0 and counts[True][2] == 1, counts
    for a, b in zip(results[True], results[False]):
        for u, v in zip(a, b):
            assert float(be.max(be.abs(u - v))) <= 1e-10 * 100


def test_grad_mode_and_oracle_engine_fall_back(torch_backend, monkeypatch):
    from oracle.aim_engines import AimDeviceMathEngine
    from oracle.oracle_engine import OracleEngine
    from optiland_b200 import plugin as P

    be = torch_backend
    eng = AimDeviceMathEngine()
    P.install(engine=eng)
    P.stats(reset=True)
    spy = _Spy(monkeypatch)
    be.grad_mode.enable()
    try:
        lens = _sample("ProjectionLens120FOV")
        lens.trace(0.0, 1.0, lens.primary_wavelength, 2, "hexapolar")
    finally:
        be.grad_mode.disable()
    assert not [c for c in eng.calls if c[0] == "aim"] and spy.subsets > 0
    assert P.stats().get("robust ray aiming: gradients wanted", 0) >= 1
    P.uninstall()
    eng = OracleEngine()
    P.install(engine=eng)
    spy = _Spy(monkeypatch)
    lens = _sample("ProjectionLens120FOV")
    lens.trace(0.0, 1.0, lens.primary_wavelength, 2, "hexapolar")
    assert spy.subsets > 0 and not any(c[0] == "aim" for c in eng.calls)


def test_failing_stop_radius_strategy_warns_once_per_solve(aim_plugin, monkeypatch):
    import warnings

    from optiland.rays.ray_aiming.initialization import RealReferenceStrategy

    P, eng, be = aim_plugin

    def broken(self):
        raise ValueError("broken on purpose")

    monkeypatch.setattr(RealReferenceStrategy, "_trace_real_marginal_ray", broken)
    counts = {}
    for device in (False, True):
        P._state["device_aim"] = device
        lens = _sample("ProjectionLens120FOV")
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            lens.trace(0.0, 0.5, lens.primary_wavelength, 2, "hexapolar")
        counts[device] = sum("RealReferenceStrategy failed" in str(w.message) for w in rec)
    assert counts[True] == counts[False] > 0, counts


# ---- GPU ---------------------------------------------------------------------------------------------------------------

def _cuda_solve(a, dtype):
    import torch

    import optiland.backend as be

    from optiland_b200.trace import DeviceTable, aim_device

    dev = torch.device("cuda:0")
    g = {k: torch.as_tensor(be.to_numpy(be.as_array_1d(v)), dtype=dtype, device=dev).contiguous().clone()
         for k, v in zip(KEYS, a["guess"])}
    n = g["x"].numel()
    g["w"] = torch.as_tensor(np.broadcast_to(be.to_numpy(be.as_array_1d(a["wl"])), (n,)).copy(), dtype=dtype, device=dev)
    Px = torch.as_tensor(be.to_numpy(a["Px"]), dtype=dtype, device=dev)
    Py = torch.as_tensor(be.to_numpy(a["Py"]), dtype=dtype, device=dev)
    dt = DeviceTable(a["table"], dev)
    st = aim_device(dt, g, Px, Py, 0, a["table"].num_surfaces, a["r_stop"], a["J"], a["it"].tol, a["it"].max_iter,
                    a["inf"])
    return {k: g[k].double().cpu().numpy() for k in KEYS}, int(st.item())


GPU_CASES = [("WideAngle170FOV", 0.25), ("WideAngle170FOV", 1.0), ("ProjectionLens160FOV", 0.6), ("finite", 1.0),
             ("tilted", 1.0), ("doe", 1.0), ("zernike", 1.0), ("zernike_range", 1.0)]


def _gpu_case_lens(be, name):
    builders = {"finite": _finite_object, "tilted": _tilted_stop, "doe": _doe_before_stop,
                "zernike": lambda b: _zernike_stop(b, 12.0), "zernike_range": lambda b: _zernike_stop(b, 5.0)}
    return builders[name](be) if name in builders else _sample(name)


@pytest.mark.gpu
@pytest.mark.parametrize("name,t", GPU_CASES)
def test_cuda_solve_matches_host_instantiation(torch_backend, name, t):
    import torch

    be = torch_backend
    lens = _gpu_case_lens(be, name)
    scale = _scale(lens)
    for f in lens.fields.get_field_coords():
        a = _aim_inputs(lens, float(f[0]), float(f[1]), t)
        host, hst, variant = _host_solve(a)
        got, st = _cuda_solve(a, torch.float64)
        assert st == hst, (name, variant, tuple(f), st, hst)
        if st == 0:
            for k in KEYS:
                assert float(np.max(np.abs(got[k] - host[k]))) <= 1e-10 * scale, (name, variant, k)
            # fp32: bounded against fp64 where it converges too
            g32, st32 = _cuda_solve(a, torch.float32)
            if st32 == 0:
                for k in ("x", "y", "L", "M"):
                    assert float(np.max(np.abs(g32[k] - host[k]))) <= 1e-3 * scale, (name, variant, k)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ROBUST)
def test_cuda_robust_trace_equals_numpy_with_one_launch_per_solve(name):
    from oracle.ref_import import import_reference

    import_reference()
    import optiland.backend as be

    from optiland_b200 import _lib
    from optiland_b200 import plugin as P

    lens0 = _sample(name)
    fields = [tuple(float(v) for v in f) for f in lens0.fields.get_field_coords()]
    want = _numpy_records(name, fields)
    be.set_backend("torch")
    be.set_precision("float64")
    be.grad_mode.disable()
    be.set_device("cuda")
    eng = P.CudaEngine()
    P.install(engine=eng)
    P.stats(reset=True)
    lib = _lib.load()
    try:
        lens = _sample(name)
        for (hx, hy), w in zip(fields, want):
            n0, l0 = len(eng.calls), lib.olb_launch_count()
            lens.trace(hx, hy, lens.primary_wavelength, 4, "hexapolar")
            launches = lib.olb_launch_count() - l0
            assert launches == len(eng.calls) - n0 and any(c[0] == "aim" for c in eng.calls[n0:]), (launches,)
            _check_records(be, lens, w, (name, hx, hy))
        assert set(P.stats()) <= {"fused launch: non-paraxial ray aiming"}, P.stats()
    finally:
        P.uninstall()
        be.set_device("cpu")
        be.set_backend("numpy")
