"""The hand-derived adjoint (olb_math.cuh::surface_backward, CPU instantiation) against central
finite differences of the NumPy oracle, on the config-3 system (reverse telephoto + 2 even
aspheres) and on a mirror system.  Loss = a random linear functional of every recorded quantity
on every surface, so every adjoint path is exercised."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from oracle import trace_oracle as O
from optiland_b200 import _lib
from optiland_b200 import table as T
from tests._util import REC, Case
from oracle.hostcheck_api import run_backward  # noqa: F401
from tests.test_hostcheck import hc  # noqa: F401  (fixture)

GP = dict(TX=0, TY=1, TZ=2, CURV=3, CONIC=4, N1=5, N2=6, COEF=7, R=19)


def loss_fn(table, rays, weights):
    _, rec, _ = O.trace(table, rays)
    return sum(float(np.sum(weights[k] * rec[k])) for k in REC)


def perturbed(table, s, **kw):
    spec = table.surfaces[s]
    ch = {}
    for k, d in kw.items():
        if k == "curv":
            ch["radius"] = 1.0 / (1.0 / spec.radius + d)
        elif k == "tz":
            t = spec.t.copy(); t[2] += d; ch["t"] = t
        elif k == "tx":
            t = spec.t.copy(); t[0] += d; ch["t"] = t
        elif k == "conic":
            ch["conic"] = spec.conic + d
        elif k == "n2":
            ch["n2"] = spec.n2 + d
        elif k == "n1":
            ch["n1"] = spec.n1 + d
        elif k.startswith("coef"):
            c = spec.coefficients.copy(); c[int(k[4:])] += d; ch["coefficients"] = c
        elif k.startswith("R"):      # one entry of the pose rotation matrix (treated as 9 independent numbers)
            R = spec.R.copy(); R[int(k[1]), int(k[2])] += d; ch["R"] = R
    return table.replace_surface(s, **ch)


def fd(table, rays, weights, s, what, h):
    return (loss_fn(perturbed(table, s, **{what: h}), rays, weights)
            - loss_fn(perturbed(table, s, **{what: -h}), rays, weights)) / (2 * h)


@pytest.mark.parametrize("name", ["telephoto_c3_tol1e-10", "hubble_c4", "cooke_c1", "tilted_fold"])
def test_adjoint_matches_finite_differences(hc, name):
    c = Case(name)
    rng = np.random.default_rng(0)
    sel = rng.choice(c.n, size=min(c.n, 64), replace=False)
    rays = {k: v[sel].copy() for k, v in c.rays.items()}
    n = sel.size
    S = c.table.num_surfaces
    # tighten Newton so the oracle is differentiable to FD accuracy
    table = T.SurfaceTable([dataclasses.replace(s, tol=1e-14) for s in c.table.surfaces], c.table.wavelengths)
    weights = {k: rng.normal(size=(S, n)) for k in REC}
    _, rec, _ = O.trace(table, rays)
    gin, gpar = run_backward(hc, table, rays, rec, weights)

    # (1) gradient w.r.t. the launch state (directional FD along a random direction)
    dirs = {k: rng.normal(size=n) for k in ("x", "y", "z", "L", "M", "N", "i", "opd")}
    scale = c.scale
    h = 1e-6  # small: a larger step pushes rays across the aperture edge (a jump in intensity)

    def shifted(sign):
        r = {k: v.copy() for k, v in rays.items()}
        r["opd"] = np.zeros(n)
        for k, d in dirs.items():
            r[k] = r[k] + sign * h * d
        return r

    fd_dir = (loss_fn(table, shifted(+1), weights) - loss_fn(table, shifted(-1), weights)) / (2 * h)
    an_dir = sum(float(np.sum(gin[k] * dirs[k])) for k in dirs)
    assert an_dir == pytest.approx(fd_dir, rel=1e-4)

    # (2) gradients w.r.t. surface parameters
    checked = 0
    for s, spec in enumerate(table.surfaces):
        if spec.kind == T.GEOM_NOOP:
            continue
        tests = [("tz", GP["TZ"], 1e-6 * scale), ("tx", GP["TX"], 1e-6 * scale), ("n1", GP["N1"], 1e-6)]
        if not spec.reflective:
            tests.append(("n2", GP["N2"], 1e-6))
        if spec.kind in (T.GEOM_STANDARD, T.GEOM_EVEN_ASPHERE) and np.isfinite(spec.radius):
            tests += [("curv", GP["CURV"], 1e-7 / max(abs(spec.radius), 1.0) ** 0), ("conic", GP["CONIC"], 1e-5)]
        if spec.kind == T.GEOM_EVEN_ASPHERE:
            tests += [(f"coef{j}", GP["COEF"] + j, 1e-6) for j in range(len(spec.coefficients))]
        if spec.rotated:             # dLoss/dR, the input of the tilt-angle gradients
            tests += [(f"R{i}{j}", GP["R"] + 3 * i + j, 1e-7) for i in range(3) for j in range(3)]
        else:
            assert not np.any(gpar[s, GP["R"]:GP["R"] + 9])
        for what, slot, hh in tests:
            if what == "curv":
                hh = 1e-5 * abs(1.0 / spec.radius)
            ref = fd(table, rays, weights, s, what, hh)
            got = gpar[s, slot]
            # n2 of surface s is n1 of surface s+1 only in a live system; here they are independent slots
            assert got == pytest.approx(ref, rel=1e-4, abs=1e-6 * np.abs(gpar).max()), (name, s, what, got, ref)
            checked += 1
    assert checked > 10


def rms_spot_and_grads(x, y):
    """loss = sqrt(mean((x-mean x)^2 + (y-mean y)^2)) (the rms_spot_size operand,
    optiland/optimization/operand/ray.py:299-342) and dloss/dx, dloss/dy."""
    n = x.size
    dx, dy = x - x.mean(), y - y.mean()
    loss = np.sqrt(np.mean(dx**2 + dy**2))
    return loss, dx / (n * loss), dy / (n * loss)


def test_config3_gradients_match_reference_autograd(hc):
    """d(RMS spot)/d(radius, conic, z) on the reverse telephoto with two even aspheres equals the
    REFERENCE's torch-CPU fp64 autograd (tests/golden/telephoto_c3_grad.npz, oracle/make_golden.py)."""
    import os

    from tests._util import GOLDEN

    c = Case("telephoto_c3_tol1e-10")
    g = np.load(os.path.join(GOLDEN, "telephoto_c3_grad.npz"))
    table = T.SurfaceTable([dataclasses.replace(s, tol=1e-14) for s in c.table.surfaces], c.table.wavelengths)
    _, rec, _ = O.trace(table, c.rays)
    loss, gx, gy = rms_spot_and_grads(rec["x"][-1], rec["y"][-1])
    assert loss == pytest.approx(float(g["loss"]), rel=1e-9)
    S, n = table.num_surfaces, c.n
    grec = {k: None for k in REC}
    grec["x"] = np.zeros((S, n)); grec["x"][-1] = gx
    grec["y"] = np.zeros((S, n)); grec["y"][-1] = gy
    _, gpar = run_backward(hc, table, c.rays, rec, grec)
    for s in (1, 2, 13):
        curv = 1.0 / table.surfaces[s].radius
        d_radius = -curv * curv * gpar[s, GP["CURV"]]
        assert d_radius == pytest.approx(float(g[f"d_radius_{s}"]), rel=1e-7), s
    for s in (1, 13):
        assert gpar[s, GP["CONIC"]] == pytest.approx(float(g[f"d_conic_{s}"]), rel=1e-7), s
    # cs.z of surface 1 is a leaf in the reference and every later surface sits at z_prev + thickness
    # (surfaces/factories/coordinate_system_factory.py:72-79): d/dz_1 shifts the whole system
    assert gpar[1:, GP["TZ"]].sum() == pytest.approx(float(g["d_z_1"]), rel=1e-7)


def test_tilt_angle_gradient_through_dLoss_dR(hc):
    """d loss / d(rx, ry, rz) of a tilted mirror: chain dLoss/dR (adjoint) with dR/d(angle) of R = Rz Ry Rx
    (coordinate_system.py:121-143) and compare with central differences of the oracle in the ANGLES."""
    c = Case("tilted_fold")
    rng = np.random.default_rng(5)
    sel = rng.choice(c.n, size=48, replace=False)
    rays = {k: v[sel].copy() for k, v in c.rays.items()}
    S, n = c.table.num_surfaces, sel.size
    weights = {k: rng.normal(size=(S, n)) for k in REC}
    s = next(j for j, sp in enumerate(c.table.surfaces) if sp.rotated)
    ang0 = np.array([0.31, -0.12, 0.07])

    def with_angles(a):
        return c.table.replace_surface(s, R=T.rotation_matrix(*a) + 0.0)

    table = with_angles(ang0)
    _, rec, _ = O.trace(table, rays)
    _, gpar = run_backward(hc, table, rays, rec, weights)
    gR = gpar[s, GP["R"]:GP["R"] + 9].reshape(3, 3)
    for q in range(3):
        h = 1e-6
        e = np.zeros(3); e[q] = h
        dR = (T.rotation_matrix(*(ang0 + e)) - T.rotation_matrix(*(ang0 - e))) / (2 * h)
        got = float(np.sum(gR * dR))
        ref = (loss_fn(with_angles(ang0 + e), rays, weights) - loss_fn(with_angles(ang0 - e), rays, weights)) / (2 * h)
        assert got == pytest.approx(ref, rel=1e-4, abs=1e-6 * np.abs(gpar).max()), (q, got, ref)


def test_odd_asphere_adjoint_matches_finite_differences(hc):
    """Odd aspheres (sag = conic + sum C_i r^(i+1), odd_asphere.py:86-142) are inside the adjoint's scope: launch
    state and parameter gradients (curvature, conic, every coefficient, pose) against central differences."""
    rng = np.random.default_rng(11)
    n = 48
    specs = [
        T.SurfaceSpec(kind=T.GEOM_NOOP),
        T.SurfaceSpec(kind=T.GEOM_ODD_ASPHERE, radius=45.0, conic=-0.3, t=[0.1, -0.05, 8.0], n1=[1.0], n2=[1.52],
                      coefficients=[0.0, 2e-4, -3e-5, 4e-6], tol=1e-14, max_iter=60),
        T.SurfaceSpec(kind=T.GEOM_ODD_ASPHERE, radius=-60.0, conic=0.2, t=[0.0, 0.0, 13.0], n1=[1.52], n2=[1.0],
                      coefficients=[1e-3, -1e-4, 2e-5], tol=1e-14, max_iter=60, R=T.rotation_matrix(0.02, -0.01, 0.3) + 0.0),
        T.SurfaceSpec(kind=T.GEOM_PLANE, t=[0.0, 0.0, 40.0]),
    ]
    table = T.SurfaceTable(specs, [0.55])
    ht = _lib.HostTable(table)
    assert hc.olbhc_bwd_supported(C.byref(ht.c)) == 1
    r = 1.0 + 4.0 * np.sqrt(rng.random(n))           # keep away from the cone tip r = 0 (C_0 r term)
    th = 2 * np.pi * rng.random(n)
    rays = dict(x=r * np.cos(th), y=r * np.sin(th), z=np.zeros(n), L=rng.normal(0, 0.02, n), M=rng.normal(0, 0.02, n),
                i=np.ones(n), w=np.full(n, 0.55))
    rays["N"] = np.sqrt(1 - rays["L"] ** 2 - rays["M"] ** 2)
    S = table.num_surfaces
    weights = {k: rng.normal(size=(S, n)) for k in REC}
    _, rec, _ = O.trace(table, rays)
    gin, gpar = run_backward(hc, table, rays, rec, weights)
    dirs = {k: rng.normal(size=n) for k in ("x", "y", "L", "M")}
    h = 1e-6

    def shifted(sign):
        rr = {k: v.copy() for k, v in rays.items()}
        for k, d in dirs.items():
            rr[k] = rr[k] + sign * h * d
        return rr

    fd_dir = (loss_fn(table, shifted(+1), weights) - loss_fn(table, shifted(-1), weights)) / (2 * h)
    an_dir = sum(float(np.sum(gin[k] * dirs[k])) for k in dirs)
    assert an_dir == pytest.approx(fd_dir, rel=1e-4)
    gmax = np.abs(gpar).max()
    for s in (1, 2):
        spec = table.surfaces[s]
        tests = [("tz", GP["TZ"], 1e-6), ("tx", GP["TX"], 1e-6), ("curv", GP["CURV"], 1e-5 * abs(1.0 / spec.radius)),
                 ("conic", GP["CONIC"], 1e-5), ("n2", GP["N2"], 1e-6)]
        tests += [(f"coef{j}", GP["COEF"] + j, 1e-7) for j in range(len(spec.coefficients))]
        for what, slot, hh in tests:
            ref = fd(table, rays, weights, s, what, hh)
            assert gpar[s, slot] == pytest.approx(ref, rel=2e-4, abs=1e-6 * gmax), (s, what, gpar[s, slot], ref)


def test_odd_asphere_adjoint_on_the_vertex_ray(hc):
    """The ray through the vertex of an odd asphere (r == 0 exactly: the chief ray of an on-axis field): the slopes x g,
    y g vanish whatever the slope factor g is, but the sag's Hessian g I does not -- at r = 0 it is the conic
    curvature plus the r^2 term's 2 C_1.  The adjoint used the forward pass's convention (polynomial part of g := 0 at
    r == 0) there and lost that term: found by the live gradient fuzz (an on-axis hexapolar bundle through a tilted odd
    asphere, 3e-4 relative on the decenter gradients against the reference's autograd and central differences)."""
    rng = np.random.default_rng(5)
    specs = [
        T.SurfaceSpec(kind=T.GEOM_NOOP),
        T.SurfaceSpec(kind=T.GEOM_ODD_ASPHERE, radius=45.0, conic=-0.3, t=[0.0, 0.0, 8.0], n1=[1.0], n2=[1.52],
                      coefficients=[0.0, 2e-3, -3e-5, 4e-6], tol=1e-14, max_iter=60),
        T.SurfaceSpec(kind=T.GEOM_PLANE, t=[0.0, 0.0, 30.0], n1=[1.52], n2=[1.52]),
    ]
    table = T.SurfaceTable(specs, [0.55])
    n = 4
    L, M = np.array([0.0, 0.05, -0.03, 0.02]), np.array([0.0, -0.02, 0.04, 0.0])
    N = np.sqrt(1 - L**2 - M**2)
    # every ray aims at the vertex (0, 0, 8) from z = 0: the intersection is at r == 0 exactly for ray 0, to rounding else
    rays = dict(x=-8.0 * L / N, y=-8.0 * M / N, z=np.zeros(n), L=L, M=M, N=N, i=np.ones(n), w=np.full(n, 0.55))
    rays["x"][0] = rays["y"][0] = 0.0
    weights = {k: rng.normal(size=(table.num_surfaces, n)) for k in REC}
    _, rec, _ = O.trace(table, rays)
    assert rec["x"][1, 0] == 0.0 and rec["y"][1, 0] == 0.0
    gin, gpar = run_backward(hc, table, rays, rec, weights)
    h = 1e-6
    for k in ("x", "y", "L", "M"):
        for r in range(n):
            def shifted(sign):
                rr = {q: v.copy() for q, v in rays.items()}
                rr[k][r] += sign * h
                if k in ("L", "M"):
                    rr["N"][r] = np.sqrt(1 - rr["L"][r] ** 2 - rr["M"][r] ** 2)
                return rr
            ref = (loss_fn(table, shifted(+1), weights) - loss_fn(table, shifted(-1), weights)) / (2 * h)
            got = gin[k][r] - (gin["N"][r] * rays[k][r] / rays["N"][r] if k in ("L", "M") else 0.0)
            assert got == pytest.approx(ref, rel=2e-5, abs=1e-7), (k, r, got, ref)
    for what, slot, hh in (("tx", GP["TX"], 1e-6), ("tz", GP["TZ"], 1e-6), ("coef1", GP["COEF"] + 1, 1e-7)):
        ref = fd(table, rays, weights, 1, what, hh)
        assert gpar[1, slot] == pytest.approx(ref, rel=2e-4, abs=1e-6 * np.abs(gpar).max()), (what, gpar[1, slot], ref)


@pytest.mark.parametrize("name", ["zernike_fringe", "zernike_noll", "misc_apertures_coatings"])
def test_polynomial_family_adjoint_matches_finite_differences(hc, name):
    """The adjoint through Zernike / polynomial surfaces (olb_trace_bwd_* with grad_tables: implicit-function theorem with the true
    sag gradient, the Hessian of the reference's slope polynomial for the normal, table gradients mapped back to the user
    coefficients): launch-state gradients, curvature / conic / pose of the freeform surface and EVERY coefficient against
    central differences of the oracle."""
    c = Case(name)
    kinds = [s.kind for s in c.table.surfaces]
    if not any(k in (T.GEOM_ZERNIKE, T.GEOM_POLYNOMIAL) for k in kinds):
        pytest.skip("no polynomial-family surface in this fixture")
    rng = np.random.default_rng(1)
    sel = rng.choice(c.n, size=min(c.n, 48), replace=False)
    rays = {k: v[sel].copy() for k, v in c.rays.items()}
    n = sel.size
    S = c.table.num_surfaces
    specs = []
    for s in c.table.surfaces:      # forward-differentiable oracle; other Newton kinds / odd features are not in these fixtures
        specs.append(dataclasses.replace(s, tol=1e-14) if s.kind in T.NEWTON_KINDS else s)
    table = T.SurfaceTable(specs, c.table.wavelengths)
    weights = {k: rng.normal(size=(S, n)) for k in REC}
    _, rec, st = O.trace(table, rays)
    assert st == 0
    gin, gpar, gtab = run_backward(hc, table, rays, rec, weights, tables=True)
    gmax = max(np.abs(gpar).max(), np.abs(gtab).max())
    # launch state
    dirs = {k: rng.normal(size=n) for k in ("x", "y", "z", "L", "M", "N", "i", "opd")}
    h = 1e-6

    def shifted(sign):
        r = {k: v.copy() for k, v in rays.items()}
        r["opd"] = np.zeros(n)
        for k, d in dirs.items():
            r[k] = r[k] + sign * h * d
        return r

    fd_dir = (loss_fn(table, shifted(+1), weights) - loss_fn(table, shifted(-1), weights)) / (2 * h)
    assert sum(float(np.sum(gin[k] * dirs[k])) for k in dirs) == pytest.approx(fd_dir, rel=2e-4)
    checked = 0
    for s, spec in enumerate(table.surfaces):
        if spec.kind not in (T.GEOM_ZERNIKE, T.GEOM_POLYNOMIAL):
            continue
        for what, slot, hh in (("tz", GP["TZ"], 1e-6), ("tx", GP["TX"], 1e-6), ("conic", GP["CONIC"], 1e-5),
                               ("curv", GP["CURV"], 1e-5 * abs(1.0 / spec.radius))):
            ref = fd(table, rays, weights, s, what, hh)
            assert gpar[s, slot] == pytest.approx(ref, rel=2e-4, abs=1e-6 * gmax), (s, what, gpar[s, slot], ref)
            checked += 1
        coefs = spec.coefficients
        if spec.kind == T.GEOM_ZERNIKE:
            W = int(max(coefs[:, 0])) + 1
            for k, (nn, mm, cN, cc) in enumerate(coefs):
                Mk = T.zernike_monomials(int(nn), int(mm), 12)
                Nk = cN / cc if cc != 0 else 1.0
                got = Nk * float(np.sum(Mk * gtab[s, 0])) + float(np.sum(Mk * gtab[s, 1]))
                hh = 1e-6

                def with_coef(delta, k=k, Nk=Nk):
                    cf = coefs.copy()
                    cf[k, 3] += delta
                    cf[k, 2] += delta * Nk
                    return table.replace_surface(s, coefficients=cf)

                ref = (loss_fn(with_coef(hh), rays, weights) - loss_fn(with_coef(-hh), rays, weights)) / (2 * hh)
                assert got == pytest.approx(ref, rel=3e-4, abs=1e-6 * gmax), (s, k, nn, mm, got, ref)
                checked += 1
        else:
            rows, cols = coefs.shape
            for i in range(rows):
                for j in range(cols):
                    got = gtab[s, 0, i, j] + gtab[s, 1, i, j]
                    hh = 1e-6

                    def with_c(delta, i=i, j=j):
                        cf = coefs.copy()
                        cf[i, j] += delta
                        return table.replace_surface(s, coefficients=cf)

                    ref = (loss_fn(with_c(hh), rays, weights) - loss_fn(with_c(-hh), rays, weights)) / (2 * hh)
                    assert got == pytest.approx(ref, rel=3e-4, abs=1e-6 * gmax), (s, i, j, got, ref)
                    checked += 1
    assert checked >= 8


def chebyshev_table():
    """The Chebyshev surface of the `cheb_biconic_toroidal` fixture (4 x 4 coefficients, norm_x != norm_y, conic base)
    in front of two plain conics (the biconic / toroidal surfaces of the fixture are outside the adjoint's scope)."""
    c = Case("cheb_biconic_toroidal")
    specs = []
    for s in c.table.surfaces:
        if s.kind in (T.GEOM_BICONIC, T.GEOM_TOROIDAL):
            s = dataclasses.replace(s, kind=T.GEOM_STANDARD, coefficients=np.zeros(0), conic=0.2)
        elif s.kind in T.NEWTON_KINDS:
            s = dataclasses.replace(s, tol=1e-14)
        specs.append(s)
    return c, T.SurfaceTable(specs, c.table.wavelengths)


def test_chebyshev_adjoint_matches_finite_differences(hc):
    """The adjoint through a Chebyshev surface: the table upload expands sum C_ij T_i(x / norm_x) T_j(y / norm_y) into ONE
    monomial table that serves sag and slopes; the reference's slope function omits the chain-rule factors 1 / norm
    (chebyshev.py:171-181), the forward pass reproduces that and the adjoint differentiates the normal AS COMPUTED while
    the intersection uses the true sag gradient.  Launch state, pose / curvature / conic and every C_ij against central
    differences of the oracle (which evaluates the reference's cos(n arccos x) form)."""
    from optiland_b200 import autograd as AG

    c, table = chebyshev_table()
    ht = _lib.HostTable(table)
    assert hc.olbhc_bwd_supported(C.byref(ht.c))
    rng = np.random.default_rng(5)
    sel = rng.choice(c.n, size=48, replace=False)
    rays = {k: v[sel].copy() for k, v in c.rays.items()}
    n = sel.size
    S = table.num_surfaces
    weights = {k: rng.normal(size=(S, n)) for k in REC}
    _, rec, st = O.trace(table, rays)
    assert st == 0 and np.isfinite(rec["x"]).all()
    gin, gpar, gtab = run_backward(hc, table, rays, rec, weights, tables=True)
    gmax = max(np.abs(gpar).max(), np.abs(gtab).max())
    dirs = {k: rng.normal(size=n) for k in ("x", "y", "z", "L", "M", "N", "i", "opd")}
    h = 1e-6

    def shifted(sign):
        r = {k: v.copy() for k, v in rays.items()}
        r["opd"] = np.zeros(n)
        for k, d in dirs.items():
            r[k] = r[k] + sign * h * d
        return r

    fd_dir = (loss_fn(table, shifted(+1), weights) - loss_fn(table, shifted(-1), weights)) / (2 * h)
    assert sum(float(np.sum(gin[k] * dirs[k])) for k in dirs) == pytest.approx(fd_dir, rel=2e-4)
    s = [j for j, sp in enumerate(table.surfaces) if sp.kind == T.GEOM_CHEBYSHEV][0]
    spec = table.surfaces[s]
    for what, slot, hh in (("tz", GP["TZ"], 1e-6), ("tx", GP["TX"], 1e-6), ("conic", GP["CONIC"], 1e-5),
                           ("curv", GP["CURV"], 1e-5 * abs(1.0 / spec.radius)), ("n2", GP["N2"], 1e-6)):
        ref = fd(table, rays, weights, s, what, hh)
        assert gpar[s, slot] == pytest.approx(ref, rel=2e-4, abs=1e-6 * gmax), (what, gpar[s, slot], ref)
    coefs = np.atleast_2d(spec.coefficients)
    K = coefs.size
    gc = AG.tables_to_coef_grads(table, gtab, K)[s].reshape(coefs.shape)
    for i in range(coefs.shape[0]):
        for j in range(coefs.shape[1]):
            def with_c(delta, i=i, j=j):
                cf = coefs.copy()
                cf[i, j] += delta
                return table.replace_surface(s, coefficients=cf)

            ref = (loss_fn(with_c(1e-6), rays, weights) - loss_fn(with_c(-1e-6), rays, weights)) / 2e-6
            assert gc[i, j] == pytest.approx(ref, rel=3e-4, abs=1e-6 * gmax), (i, j, gc[i, j], ref)


def test_forbes_qbfs_adjoint_matches_finite_differences(hc):
    """The adjoint through Forbes Q^bfs surfaces (forbes/geometry.py:187-366): slope factor and its r^2-derivative from the
    Clenshaw sum with two derivatives, curvature / conic entering the departure through phi, coefficient gradients in the
    Clenshaw basis mapped back to the user's a_m by the transposed change of basis (``autograd.forbes_basis_matrix``).
    Launch state, pose, curvature, conic and every a_m of both surfaces of the `forbes_qbfs` fixture (conic -0.4 and 0,
    6 and 5 terms) against central differences of the oracle."""
    from optiland_b200 import autograd as AG

    c = Case("forbes_qbfs")
    table = T.SurfaceTable([dataclasses.replace(s, tol=1e-14) if s.kind in T.NEWTON_KINDS else s for s in c.table.surfaces],
                           c.table.wavelengths)
    ht = _lib.HostTable(table)
    assert hc.olbhc_bwd_supported(C.byref(ht.c))
    rng = np.random.default_rng(7)
    sel = rng.choice(c.n, size=48, replace=False)
    rays = {k: v[sel].copy() for k, v in c.rays.items()}
    n = sel.size
    S = table.num_surfaces
    weights = {k: rng.normal(size=(S, n)) for k in REC}
    _, rec, st = O.trace(table, rays)
    assert st == 0 and np.isfinite(rec["x"]).all()
    gin, gpar, gtab = run_backward(hc, table, rays, rec, weights, tables=True)
    gmax = np.abs(gpar).max()
    dirs = {k: rng.normal(size=n) for k in ("x", "y", "z", "L", "M", "N", "i", "opd")}
    h = 1e-6

    def shifted(sign):
        r = {k: v.copy() for k, v in rays.items()}
        r["opd"] = np.zeros(n)
        for k, d in dirs.items():
            r[k] = r[k] + sign * h * d
        return r

    fd_dir = (loss_fn(table, shifted(+1), weights) - loss_fn(table, shifted(-1), weights)) / (2 * h)
    assert sum(float(np.sum(gin[k] * dirs[k])) for k in dirs) == pytest.approx(fd_dir, rel=2e-4)
    checked = 0
    for s, spec in enumerate(table.surfaces):
        if spec.kind != T.GEOM_FORBES_QBFS:
            continue
        for what, slot, hh in (("tz", GP["TZ"], 1e-6), ("tx", GP["TX"], 1e-6), ("conic", GP["CONIC"], 1e-5),
                               ("curv", GP["CURV"], 1e-5 * abs(1.0 / spec.radius)), ("n2", GP["N2"], 1e-6)):
            ref = fd(table, rays, weights, s, what, hh)
            assert gpar[s, slot] == pytest.approx(ref, rel=2e-4, abs=1e-6 * gmax), (s, what, gpar[s, slot], ref)
            checked += 1
        nc = len(spec.coefficients)
        ga = AG.forbes_coef_grads(gpar[s, GP["COEF"]:GP["COEF"] + nc])
        for m in range(nc):
            ref = fd(table, rays, weights, s, f"coef{m}", 1e-6)
            assert ga[m] == pytest.approx(ref, rel=3e-4, abs=1e-6 * gmax), (s, m, ga[m], ref)
            checked += 1
    assert checked == 2 * 5 + 6 + 5
