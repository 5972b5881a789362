"""BASELINE.json's configurations at their STATED shapes (fixtures `*_ref.npz` / `*_grad.npz` written by
oracle/make_golden.py::case_config_shapes / case_c3_grad_full_size from the unmodified reference):

* config 1: Cooke triplet, 3 fields x 1 wavelength, hexapolar pupil with 64 rings (12 481 points per field): the
  reference's SpotDiagram RMS radii;
* config 3: d(RMS spot)/d(radius, conic, z) over the full 1 154-ring hexapolar pupil (3 998 611 rays) against the
  reference's own torch-CPU autograd (accumulated over chunks);
* config 5: Zernike + Fresnel + PolarizedRays, 5 fields x 3 wavelengths: every OPD MAP (reference `Wavefront`, chief-ray
  strategy) within 1e-5 waves, plus the trace_generic call shape with P matrices.

`-m "not gpu"`: the oracle (and the CPU instantiation of the device math) against the fixtures; `-m gpu`: the kernels.
"""
import os

import numpy as np
import pytest

from optiland_b200 import table as T
from optiland_b200.launch import launch_from_affine, pupil_affine, pupil_affine_fields
from optiland_b200.table import SurfaceTable
from tests._util import GOLDEN, Case


def hexapolar(num_rings):
    """optiland/distribution.py HexagonalDistribution.generate_points (:196-220): centre + 6 i points on ring i."""
    x, y = [np.zeros(1)], [np.zeros(1)]
    r = np.linspace(0, 1, num_rings + 1)
    for i in range(num_rings):
        th = np.linspace(0, 2 * np.pi, 6 * (i + 1) + 1)[:-1]
        x.append(r[i + 1] * np.cos(th))
        y.append(r[i + 1] * np.sin(th))
    return np.concatenate(x), np.concatenate(y)


# --------------------------------------------------------------------------- config 1
def _c1():
    z = np.load(os.path.join(GOLDEN, "c1_cooke_64rings_ref.npz"), allow_pickle=False)
    table = SurfaceTable.from_arrays(z)
    scs = [{k[len(f"f{j}_launch_"):]: float(z[k]) for k in z.files if k.startswith(f"f{j}_launch_")} for j in range(3)]
    return z, table, scs


def _rms_about(x, y, inten, center):
    m = inten > 0
    return float(np.sqrt(np.mean((x[m] - center[0]) ** 2 + (y[m] - center[1]) ** 2)))


def test_hexapolar_helper_matches_the_fixture_size():
    z, _, _ = _c1()
    Px, _ = hexapolar(int(z["n_rings"]))
    assert Px.size == int(z["n_pupil"]) == 12481


def test_config1_64_rings_oracle_reproduces_reference_spot_radii():
    from oracle import trace_oracle as O

    z, table, scs = _c1()
    Px, Py = hexapolar(64)
    for j, sc in enumerate(scs):
        x, y, zz, L, M, N = launch_from_affine(Px, Py, pupil_affine(sc))
        fin, rec, _ = O.trace(table, dict(x=x, y=y, z=zz, L=L, M=M, N=N, i=np.ones_like(x), w=np.full_like(x, 0.55)))
        # image plane is untilted at z = const: local (x, y) == global (x, y)
        rms = _rms_about(rec["x"][-1], rec["y"][-1], rec["intensity"][-1], z["chief_center"][j])
        assert rms == pytest.approx(float(z["spot_rms"][j, 0]), rel=1e-10)
        m = rec["intensity"][-1] > 0
        cen = (rec["x"][-1][m].mean(), rec["y"][-1][m].mean())
        assert _rms_about(rec["x"][-1], rec["y"][-1], rec["intensity"][-1], cen) == pytest.approx(float(z["spot_rms_centroid"][j, 0]), rel=1e-10)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
def test_config1_64_rings_kernel_spot_radii(dtype_name):
    """Config 1 at its stated shape on the GPU: records path (what SpotDiagram reads) and the fused moments epilogue."""
    import torch

    from optiland_b200.trace import DeviceTable, moments_to_spot, trace_moments_device, trace_pupil_device

    dtype = getattr(torch, dtype_name)
    z, table, scs = _c1()
    Px, Py = hexapolar(64)
    dPx, dPy = torch.from_numpy(Px).to("cuda", dtype), torch.from_numpy(Py).to("cuda", dtype)
    dtab = DeviceTable(table)
    rel = 1e-9 if dtype == torch.float64 else 2e-3       # fp32: 4-15 um spots from intercepts good to ~1e-5 mm
    for j, sc in enumerate(scs):
        aff = pupil_affine(sc)
        rays, rec = trace_pupil_device(dtab, dPx, dPy, aff, 0, table.num_surfaces)
        x, y, inten = (rec[k][-1].double().cpu().numpy() for k in ("x", "y", "intensity"))
        assert _rms_about(x, y, inten, z["chief_center"][j]) == pytest.approx(float(z["spot_rms"][j, 0]), rel=rel)
        cen = z["chief_center"][j]
        mom = trace_moments_device(dtab, Px.size, dtype, pupil=(dPx, dPy, aff), center=(float(cen[0]), float(cen[1])))
        sp = moments_to_spot(mom, (float(cen[0]), float(cen[1])))
        assert sp["count"] == Px.size
        assert sp["rms_center"] == pytest.approx(float(z["spot_rms"][j, 0]), rel=rel)
        assert sp["rms_centroid"] == pytest.approx(float(z["spot_rms_centroid"][j, 0]), rel=rel)


# --------------------------------------------------------------------------- config 5
def _c5():
    z = np.load(os.path.join(GOLDEN, "c5_opd_maps_ref.npz"), allow_pickle=False)
    tables = [SurfaceTable.from_arrays(z, prefix=f"w{wi}_tab_") for wi in range(3)]
    return z, tables


def _c5_case(z, fi, wi):
    tag = f"f{fi}w{wi}"
    sc = {k[len(tag) + 8:]: float(z[k]) for k in z.files if k.startswith(f"{tag}_launch_")}
    ref = {k: (np.array(z[f"{tag}_ref_{k}"]) if k in ("center", "tilt") else float(z[f"{tag}_ref_{k}"]))
           for k in ("center", "radius", "n_image", "tilt", "opd_ref", "wavelength_um")}
    want = {k: np.array(z[f"{tag}_{k}"]) for k in ("opd", "pupil_x", "pupil_y", "pupil_z", "intensity", "p")}
    return sc, ref, want


def test_config5_opd_maps_oracle_vs_reference():
    from oracle import trace_oracle as O

    z, tables = _c5()
    Px, Py = z["Px"], z["Py"]
    for fi in range(5):
        for wi in range(3):
            sc, ref, want = _c5_case(z, fi, wi)
            x, y, zz, L, M, N = launch_from_affine(Px, Py, pupil_affine(sc))
            inp = dict(x=x, y=y, z=zz, L=L, M=M, N=N, i=np.ones_like(x), w=np.full_like(x, ref["wavelength_um"]),
                       p=np.tile(np.eye(3, dtype=np.complex128), (x.size, 1, 1)))
            fin, rec, _ = O.trace(tables[wi], inp, polarized=True)
            got = O.wavefront_reference_sphere(fin, Px, Py, ref)
            assert np.max(np.abs(got["opd"] - want["opd"])) <= 1e-6, (fi, wi)       # waves
            assert np.max(np.abs(fin["p"] - want["p"])) <= 1e-12
            np.testing.assert_allclose(got["intensity"], want["intensity"], atol=1e-13)


@pytest.mark.gpu
def test_config5_opd_maps_kernel_within_1e5_waves():
    """BASELINE.json config 5's tolerance, map by map, 5 fields x 3 wavelengths, through olb_trace_call_f64, polarized (pupil
    launch + P matrices in shared memory + wavefront epilogue)."""
    import torch

    from optiland_b200.trace import DeviceTable, trace_wavefront_device

    z, tables = _c5()
    Px = torch.from_numpy(z["Px"]).to("cuda", torch.float64)
    Py = torch.from_numpy(z["Py"]).to("cuda", torch.float64)
    worst = 0.0
    for wi in range(3):
        dtab = DeviceTable(tables[wi])
        for fi in range(5):
            sc, ref, want = _c5_case(z, fi, wi)
            got = trace_wavefront_device(dtab, Px, Py, pupil_affine(sc), ref, polarized=True)
            err = float(np.max(np.abs(got["opd"].cpu().numpy() - want["opd"])))
            worst = max(worst, err)
            assert err <= 1e-5, (fi, wi, err)
            for k in ("pupil_x", "pupil_y", "pupil_z"):
                assert np.max(np.abs(got[k].cpu().numpy() - want[k])) <= 1e-10 * ref["radius"]
            assert np.max(np.abs(got["intensity"].cpu().numpy() - want["intensity"])) <= 1e-12
            assert np.max(np.abs(got["p"].cpu().numpy() - want["p"])) <= 1e-11
    print(f"config 5: worst OPD-map error over 15 maps {worst:.2e} waves")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
def test_config5_generic_polarized_pupil_launch(dtype_name):
    """trace_generic's call shape with PolarizedRays through the fused launch (per-ray fields and wavelengths, P
    starting as the identity in-kernel) against the reference's records and P matrices."""
    import torch

    from optiland_b200.trace import DeviceTable, trace_pupil_device

    dtype = getattr(torch, dtype_name)
    c = Case("generic_polarized_c5")
    sc = {k[9:]: float(c.z[k]) for k in c.z.files if k.startswith("x_launch_")}
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dtype)  # noqa: E731
    aff = pupil_affine_fields(sc, dev(c.extra("Hx")), dev(c.extra("Hy")))
    rays, rec = trace_pupil_device(DeviceTable(c.table), dev(c.extra("Px")), dev(c.extra("Py")), aff, 0,
                                   c.table.num_surfaces, wavelength=dev(c.rays["w"]), polarization="matrix")
    f64 = dtype == torch.float64
    tol = 1e-11 * c.scale + 2e-10 if f64 else 3e-6 * c.scale
    for k in ("x", "y", "z", "opd"):
        got = rec[k].double().cpu().numpy()
        assert np.max(np.abs(got - c.rec[k])) <= tol, k
    assert np.max(np.abs(rays.p.cpu().numpy().astype(np.complex128) - c.out["p"])) <= (1e-11 if f64 else 2e-5)
    assert np.max(np.abs(rays.i.double().cpu().numpy() - c.rec["intensity"][-1])) <= 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["zernike_polarized_c5", "cooke_polarized", "tilted_fold_polarized"])
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
def test_intensity_epilogue_in_kernel(name, dtype_name):
    """PolarizedRays.update_intensity as the kernel's epilogue (OlbTraceCall.pol): rays.i against the reference's
    value; the record rows keep the geometric intensity."""
    import torch

    from optiland_b200.trace import DeviceTable, PolarizedRays, trace_device

    dtype = getattr(torch, dtype_name)
    c = Case(name)
    r = c.rays
    state = tuple(c.extra("state")) if "x_state" in c.z else None
    want = c.extra("final_intensity") if state is not None else c.extra("final_intensity_unpolarized")
    rays = PolarizedRays(r["x"], r["y"], r["z"], r["L"], r["M"], r["N"], r["i"], r["w"], dtype=dtype)
    rec = trace_device(DeviceTable(c.table), rays, 0, c.table.num_surfaces, polarization=state)
    f64 = dtype == torch.float64
    assert np.max(np.abs(rays.i.double().cpu().numpy() - want)) <= (1e-11 if f64 else 5e-5)
    assert np.max(np.abs(rec["intensity"].double().cpu().numpy() - c.rec["intensity"])) <= (1e-12 if f64 else 1e-6)
    assert np.max(np.abs(rays.p.cpu().numpy().astype(np.complex128) - c.out["p"])) <= (1e-11 if f64 else 2e-5)


# --------------------------------------------------------------------------- config 3
@pytest.mark.gpu
def test_config3_gradient_at_full_size_4M_rays():
    """Config 3's autograd check at its stated size: the adjoint kernel over the 3 998 611-ray hexapolar pupil against
    the reference's own torch-CPU fp64 autograd (fixture: accumulated over chunks)."""
    import torch

    from optiland_b200.autograd import GP_CONIC, GP_CURV, GP_TZ, table_to_params, trace_differentiable
    from optiland_b200.trace import RealRays

    path = os.path.join(GOLDEN, "telephoto_c3_4M_grad.npz")
    if not os.path.exists(path):
        pytest.skip("fixture not generated (oracle/make_golden.py c3full)")
    g = np.load(path)
    c = Case("telephoto_c3_tol1e-10")
    sc = {"EPL": float(g["launch_EPL"]), "EPD": float(g["launch_EPD"]), "offset": float(g["launch_offset"]),
          "max_field": float(g["launch_max_field"]), "z1": float(g["launch_z1"]), "vx": 1.0, "vy": 1.0, "Hx": 0.0, "Hy": 0.7}
    Px, Py = hexapolar(int(g["n_rings"]))
    assert Px.size == int(g["n_rays"])
    x, y, z, L, M, N = launch_from_affine(torch.from_numpy(Px).cuda(), torch.from_numpy(Py).cuda(), pupil_affine(sc))
    rays = RealRays(x, y, z, L, M, N, 1.0, 0.5876, dtype=torch.float64)
    params = table_to_params(c.table).cuda().requires_grad_(True)
    rec = trace_differentiable(c.table, params, rays, rows=(-1,))
    xs, ys = rec["x"], rec["y"]
    loss = torch.sqrt(torch.mean((xs - xs.mean()) ** 2 + (ys - ys.mean()) ** 2))
    loss.backward()
    gp = params.grad.cpu().numpy()
    p = params.detach().cpu().numpy()
    assert float(loss) == pytest.approx(float(g["loss"]), rel=1e-9)
    for s in (1, 2, 13):
        # d/d radius = -curv^2 d/d curv
        assert -p[s, GP_CURV] ** 2 * gp[s, GP_CURV] == pytest.approx(float(g[f"d_radius_{s}"]), rel=2e-6), s
    for s in (1, 13):
        assert gp[s, GP_CONIC] == pytest.approx(float(g[f"d_conic_{s}"]), rel=2e-6, abs=1e-12), s
        # the reference chains the vertex positions: surface s's cs.z is a leaf that every later surface's z is
        # built from (thickness-based construction), so its gradient is the sum over the surfaces behind it
        assert gp[s:, GP_TZ].sum() == pytest.approx(float(g[f"d_z_{s}"]), rel=2e-6, abs=1e-12), s
