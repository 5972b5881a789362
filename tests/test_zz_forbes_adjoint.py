"""Forbes Q^bfs surfaces in the adjoint (olb_math.cuh::surface_backward, the Forbes branch).

The branch was written after most of the round's GPU budget had been spent, which is why these tests sit in a file of
their own that sorts last; the final minute of the budget then ran them on the GPU (``profiles/r2b_gputests_forbes.log``:
the kernel in fp64 and fp32 against the CPU instantiation of the same adjoint, and the plugin path on the product engine
against the reference's own eager autograd -- 3 passed).  CPU side: finite differences of the oracle in
tests/test_hostcheck_backward.py, and the plugin path over the test-only oracle engine, below."""
import dataclasses

import numpy as np
import pytest

from oracle.ref_import import reference_available
from tests._util import REC, Case
from tests.test_plugin_reference import plugin  # noqa: F401  (fixture: [oracle] on CPU, [cuda] on the GPU)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
def test_forbes_adjoint_kernel_matches_cpu_instantiation(dtype_name):
    """olb_trace_bwd_* with grad_tables on a table with two Forbes Q^bfs surfaces (the `forbes_qbfs` fixture): gradients of a random
    linear functional of all records w.r.t. the launch state and every surface parameter -- the coefficient slots hold
    dLoss/db_m (Clenshaw basis), mapped to the user's a_m by ``_TraceFn.backward`` -- against the CPU instantiation of the
    same adjoint, which tests/test_hostcheck_backward.py holds to finite differences of the oracle."""
    import torch

    from oracle import trace_oracle as O
    from oracle.hostcheck_api import load, run_backward
    from optiland_b200 import autograd as AG
    from optiland_b200 import table as T
    from optiland_b200.trace import RealRays

    c = Case("forbes_qbfs")
    rng = np.random.default_rng(11)
    n = 256
    sel = rng.choice(c.n, size=n, replace=False)
    rays_np = {k: v[sel].copy() for k, v in c.rays.items()}
    table = T.SurfaceTable([dataclasses.replace(s, tol=1e-13) if s.kind in T.NEWTON_KINDS else s for s in c.table.surfaces],
                           c.table.wavelengths)
    S = table.num_surfaces
    w = {k: rng.normal(size=(S, n)) for k in REC}
    _, rec, _ = O.trace(table, rays_np)
    gin, gpar, _ = run_backward(load(), table, rays_np, rec, w, tables=True)
    for s, spec in enumerate(table.surfaces):
        if spec.kind == T.GEOM_FORBES_QBFS:
            nc = len(spec.coefficients)
            gpar[s, AG.GP_COEF:AG.GP_COEF + nc] = AG.forbes_coef_grads(gpar[s, AG.GP_COEF:AG.GP_COEF + nc])
    dtype = getattr(torch, dtype_name)
    params = AG.table_to_params(table).cuda().requires_grad_(True)
    rr = RealRays(*[rays_np[k] for k in ("x", "y", "z", "L", "M", "N", "i", "w")], dtype=dtype)
    for k in ("x", "y", "L"):
        getattr(rr, k).requires_grad_(True)
    out = AG.trace_differentiable(table, params, rr)
    loss = sum((out[k].double() * torch.from_numpy(w[k]).cuda()).sum() for k in REC)
    loss.backward()
    gp = params.grad.cpu().numpy()
    scale = np.abs(gpar).max()
    tol = 1e-8 if dtype == torch.float64 else 2e-2
    assert np.abs(gp[:, AG.GP_COEF:AG.GP_COEF + 6]).max() > 0
    assert np.max(np.abs(gp - gpar)) <= tol * scale
    for k in ("x", "y", "L"):
        g = getattr(rr, k).grad.double().cpu().numpy()
        assert np.max(np.abs(g - gin[k])) <= tol * max(1.0, np.abs(gin[k]).max())


@pytest.mark.skipif(not reference_available(), reason="reference not present on this box")
def test_autograd_forbes_qbfs_coefficient_variables(plugin):
    """Forbes Q^bfs surfaces with be.grad_mode on: d(RMS spot + OPD)/d(a_n) for the radial terms set the way
    ForbesQNormalSlopeCoeffVariable sets them (optimization/variable/forbes_coeff.py: ``geom.radial_terms[n] = value``),
    d/d(radius), d/d(conic) -- forward kernel + the adjoint's Forbes branch (Clenshaw sum with two derivatives, gradients
    in the Clenshaw basis mapped back through the transposed change of basis) -- equal the reference's own eager autograd
    through its functional Clenshaw recurrences (forbes/qpoly.py) and unrolled Newton iterations."""
    import torch

    P, eng, be = plugin
    from optiland import optic as _optic

    def make():
        lens = _optic.Optic()
        lens.surfaces.add(index=0, radius=be.inf, thickness=be.inf)
        lens.surfaces.add(index=1, radius=22.0, thickness=6.0, material="N-BK7", is_stop=True, conic=-0.4,
                          radial_terms={0: 0.12, 1: -0.041, 2: 0.013, 3: -0.006, 5: 0.002}, norm_radius=9.0,
                          surface_type="forbes_qbfs", tol=1e-12)
        lens.surfaces.add(index=2, radius=-31.0, thickness=28.0, conic=0.0,
                          radial_terms={0: -0.27, 1: 0.087, 2: -0.048}, norm_radius=8.5,
                          surface_type="forbes_qbfs", tol=1e-12)
        lens.surfaces.add(index=3)
        lens.set_aperture(aperture_type="EPD", value=12.0)
        lens.fields.set_type(field_type="angle")
        lens.fields.add(y=0)
        lens.fields.add(y=4)
        lens.wavelengths.add(value=0.55, is_primary=True)
        return lens

    def run():
        lens = make()
        g1, g2 = lens.surfaces.surfaces[1].geometry, lens.surfaces.surfaces[2].geometry
        lens.trace(0.0, 0.7, 0.55, 6, "hexapolar")
        x, y = lens.surfaces.x[-1, :], lens.surfaces.y[-1, :]
        loss = torch.sqrt(torch.mean((x - torch.mean(x)) ** 2 + (y - torch.mean(y)) ** 2)) + 1e-3 * torch.mean(lens.surfaces.opd[-1, :])
        loss.backward()
        out = {"loss": float(loss.detach()), "radius1": float(g1.radius.grad), "conic1": float(g1.k.grad),
               "radius2": float(g2.radius.grad)}
        for name, g in (("s1", g1), ("s2", g2)):
            for n_, t in g.radial_terms.items():
                out[f"{name}.a{n_}"] = float(t.grad)
        return out

    be.grad_mode.enable()
    try:
        n0 = len(eng.calls)
        P.stats(reset=True)
        got = run()
        assert any(c[0] == "grad" for c in eng.calls[n0:]) and not P.stats(), (eng.calls[n0:], P.stats())
        P.uninstall()                       # the reference's own eager graph
        ref = run()
    finally:
        be.grad_mode.disable()
    assert got["loss"] == pytest.approx(ref["loss"], rel=1e-9)
    assert set(got) == set(ref) and len(ref) == 4 + 5 + 3
    scale = max(abs(v) for k, v in ref.items() if k != "loss")
    for k in ref:
        assert got[k] == pytest.approx(ref[k], rel=5e-6, abs=1e-8 * scale), (k, got[k], ref[k])
