"""The C-ABI shared library loads and exports every symbol include/olb.h declares (no compute)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from optiland_b200 import _lib
from optiland_b200 import table as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "olb.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(olb_[a-z0-9_]+)\s*\(", src)))


def test_header_and_binding_agree():
    assert _declared_symbols() == sorted(_lib.SYMBOLS)


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    for name in _declared_symbols():
        assert hasattr(lib, name), name
    assert lib.olb_version() >= 1


def test_struct_sizes_match_header():
    assert T.OLB_SURFACE_DTYPE.itemsize == 192
    assert C.sizeof(_lib.OlbRays) == 13 * 8
    assert C.sizeof(_lib.OlbRecords) == 9 * 8
    assert C.sizeof(_lib.OlbTable) == 40
    assert C.sizeof(_lib.OlbDeviceTable) == 72
    assert C.sizeof(_lib.OlbTraceCall) == 112


def test_table_validation_errors_no_gpu_needed():
    """olb_table_workspace_bytes validates on the host: malformed tables are rejected with a
    message, well-formed ones report a size (no device call is made)."""
    lib = _lib.load()
    good = T.SurfaceTable([T.SurfaceSpec(kind=T.GEOM_NOOP), T.SurfaceSpec(kind=T.GEOM_STANDARD, radius=50.0,
                                                                             n2=[1.5])], [0.55])
    ht = _lib.HostTable(good)
    assert lib.olb_table_workspace_bytes(C.byref(ht.c)) > 0
    ht.surf["kind"][1] = 99
    assert lib.olb_table_workspace_bytes(C.byref(ht.c)) == -5
    assert "kind" in _lib.last_error()
    ht = _lib.HostTable(good)
    ht.surf["media_off"][1] = 10_000
    assert lib.olb_table_workspace_bytes(C.byref(ht.c)) == -5
    assert "media" in _lib.last_error()


def test_pack_roundtrip():
    s = T.SurfaceSpec(kind=T.GEOM_ZERNIKE, radius=30.0, conic=-1.0, norm_radius=5.0,
                      coefficients=np.array([[2, 0, 1e-3, 5e-4], [3, -1, 2e-3, 1e-3]]),
                      aperture=T.aperture_combine(T.AP_UNION, T.aperture_radial(3.0, 1.0), T.aperture_rect(-1, 1, -2, 2)),
                      n1=[1.0, 1.0], n2=[1.5, 1.6], k1=[0.0, 1e-6], reflective=False,
                      coating=T.COAT_FRESNEL, coat_n1=[1.0, 1.0], coat_n2=[1.5, 1.6])
    tab = T.SurfaceTable([T.SurfaceSpec(kind=T.GEOM_NOOP, n1=[1, 1], n2=[1, 1], k1=[0, 0]), s], [0.5, 0.6])
    back = T.SurfaceTable.from_arrays(tab.to_arrays())
    b = back.surfaces[1]
    assert b.kind == s.kind and b.radius == s.radius and b.norm_radius == s.norm_radius
    np.testing.assert_array_equal(b.coefficients, s.coefficients)
    np.testing.assert_array_equal(b.aperture, s.aperture)
    np.testing.assert_array_equal(b.n2, s.n2)
    np.testing.assert_array_equal(b.coat_n2, s.coat_n2)
    with pytest.raises(ValueError):
        T.validate_aperture_program(np.array([T.AP_UNION], dtype=float))


def test_pupil_affine_launch_equals_reference_launch_arrays():
    """The affine (Px, Py) -> launch state form handed to the kernel reproduces the launch arrays the
    reference's RayGenerator produced (golden inputs)."""
    from optiland_b200.launch import launch_infinite_angle, pupil_affine_infinite_angle
    from tests._util import Case

    for name in ("dgauss_c2", "hubble_c4"):
        c = Case(name)
        sc = {k[9:]: float(c.z[k]) for k in c.z.files if k.startswith("x_launch_")}
        Px, Py = c.extra("Px"), c.extra("Py")
        a = pupil_affine_infinite_angle(sc)
        x0 = a["origin0"][0] + a["origin_scale"][0] * Px
        y0 = a["origin0"][1] + a["origin_scale"][1] * Py
        d = np.stack([a["target0"][0] + a["target_scale"][0] * Px - x0, a["target0"][1] + a["target_scale"][1] * Py - y0,
                      np.full_like(Px, a["target0"][2] - a["origin0"][2])])
        d /= np.linalg.norm(d, axis=0)
        ref = launch_infinite_angle(Px, Py, sc)
        for got, want, key in zip((x0, y0, d[0], d[1], d[2]), (ref[0], ref[1], ref[3], ref[4], ref[5]), "xyLMN"):
            np.testing.assert_allclose(got, want, rtol=0, atol=1e-12 * c.scale)
            np.testing.assert_allclose(got, c.rays[key], rtol=0, atol=1e-12 * c.scale)


LAUNCH_CASES = ["dgauss_c2", "hubble_c4", "finite_object_height", "finite_object_angle", "litho_telecentric"]


@pytest.mark.parametrize("name", LAUNCH_CASES)
def test_every_launch_mode_reproduces_the_reference_ray_generator(name):
    """f-1 for all launch modes (infinite-object angle field; finite object with object-height / angle
    fields; object-space telecentric): the affine form the kernel evaluates, restated by
    launch.launch_from_affine, equals the launch rays RayGenerator + ParaxialRayAimer produced."""
    from optiland_b200.launch import launch_from_affine, pupil_affine
    from tests._util import Case

    c = Case(name)
    sc = {k[9:]: float(c.z[k]) for k in c.z.files if k.startswith("x_launch_")}
    aff = pupil_affine(sc)
    got = launch_from_affine(c.extra("Px"), c.extra("Py"), aff)
    for g, key in zip(got, "xyzLMN"):
        np.testing.assert_allclose(g, c.rays[key], rtol=0, atol=1e-12 * c.scale, err_msg=key)
    if int(sc.get("mode", 0)) != 0:
        assert aff["origin_scale"] == (0.0, 0.0)      # every ray starts at the object point


GENERIC_CASES = ["generic_dgauss", "generic_finite_height", "generic_finite_angle", "generic_litho"]


@pytest.mark.parametrize("name", GENERIC_CASES)
def test_per_ray_field_launch_reproduces_trace_generic_rays(name):
    """trace_generic-shaped batches: with per-ray field arrays the launch form (launch.pupil_affine_fields, scalars
    of the H = 0 field) equals the rays RayGenerator + ParaxialRayAimer produced for (Hx, Hy, Px, Py) arrays."""
    from optiland_b200.launch import launch_from_affine, pupil_affine_fields
    from tests._util import Case

    c = Case(name)
    sc = {k[9:]: float(c.z[k]) for k in c.z.files if k.startswith("x_launch_")}
    aff = pupil_affine_fields(sc, c.extra("Hx"), c.extra("Hy"))
    got = launch_from_affine(c.extra("Px"), c.extra("Py"), aff)
    for g, key in zip(got, "xyzLMN"):
        np.testing.assert_allclose(g, c.rays[key], rtol=0, atol=1e-12 * c.scale, err_msg=key)
