"""TEST INFRASTRUCTURE ONLY -- CPU restatement (NumPy, fp64) of Optiland's ruled grating: ``DiffractiveInteractionModel``
(optiland/interactions/diffractive_model.py:28-61) on a ``PlaneGrating`` or a ``StandardGratingGeometry``, on top of
the NumPy oracle of phase-profile tables (``oracle/phase_oracle.py``), so that a table may hold both.

``trace`` has the signature and the results of ``trace_oracle.trace``.  Runs of other surfaces go through
``phase_oracle.trace`` unchanged; a grating surface is traced there with its interaction and coating taken off
(localize, distance, propagation, OPD, absorption and aperture are those of Plane / StandardGeometry), and the
diffraction and the coating step are applied here, in the surface's local frame.

The diffraction is the vector form of include/olb.h (OLB_INTERACT_GRATING), with the normal n aligned with the ray:
    a = n1 d0 + g f,  g = m lambda sqrt(fx^2 + fy^2) / d,  T = a |n|^2 - (a . n) n,  Q = n2^2 |n|^2 - |a x n|^2
    d' = normalise(+-T + sign(d) sqrt(Q) n)   (+ transmission, - reflection)
It is the reference's expanded expression (RealRays.gratingdiffract) divided through by the projected period.
"""
from __future__ import annotations

import dataclasses

import numpy as np

from oracle import phase_oracle as PO
from oracle import trace_oracle as O
from optiland_b200 import table as T


def grating_vector(s: T.SurfaceSpec, x, y, nx, ny, nz):
    """The grating vector f at the local points (x, y) with the geometry's unaligned normal n."""
    a = s.grating_angle
    if s.kind == T.GEOM_PLANE:
        return np.full_like(x, -np.sin(a)), np.full_like(x, np.cos(a)), np.zeros_like(x)
    # the groove tangent: (1, tan a) in x-y, its z slope the conic's derivative along that direction
    R, k = s.radius, s.conic
    root = np.sqrt(1.0 - (1.0 + k) * (x**2 + y**2) / R**2)
    tx, ty, tz = np.ones_like(x), np.full_like(x, np.tan(a)), (x + y * np.tan(a)) / (R * root)
    cx, cy, cz = ny * tz - nz * ty, nz * tx - nx * tz, nx * ty - ny * tx
    mag = np.sqrt(cx**2 + cy**2 + cz**2)
    return -cx / mag, -cy / mag, -cz / mag


def grating_diffraction(s: T.SurfaceSpec, L, M, N, n1, n2, w, nx, ny, nz, fx, fy, fz):
    """The diffracted direction (L, M, N); NaN for an evanescent order, as in the reference."""
    dot = L * nx + M * ny + N * nz
    sg = np.sign(dot)
    mx, my, mz = nx * sg, ny * sg, nz * sg
    g = s.grating_order * w * np.sqrt(fx**2 + fy**2) / s.grating_period
    ax, ay, az = n1 * L + g * fx, n1 * M + g * fy, n1 * N + g * fz
    nn = mx**2 + my**2 + mz**2
    adn = ax * mx + ay * my + az * mz
    Tx, Ty, Tz = ax * nn - adn * mx, ay * nn - adn * my, az * nn - adn * mz
    cx, cy, cz = ay * mz - az * my, az * mx - ax * mz, ax * my - ay * mx
    Q = n2**2 * nn - (cx**2 + cy**2 + cz**2)
    root = np.sign(s.grating_period) * np.sqrt(Q)
    sv = -1.0 if s.reflective else 1.0
    vx, vy, vz = sv * Tx + root * mx, sv * Ty + root * my, sv * Tz + root * mz
    mag = np.sqrt(vx**2 + vy**2 + vz**2)
    return vx / mag, vy / mag, vz / mag


def _grating_surface(table, si, state, P):
    """One grating surface: (state after it, status, P)."""
    s = table.surfaces[si]
    bare = dataclasses.replace(s, interaction=T.INTERACT_REFRACT, coating=T.COAT_NONE, coat_n1=None, coat_n2=None,
                               record=True)
    surfaces = list(table.surfaces)
    surfaces[si] = bare
    out, _, status = O.trace(T.SurfaceTable(surfaces, table.wavelengths), state, si, si + 1)
    x, y, z = out["x"] - s.t[0], out["y"] - s.t[1], out["z"] - s.t[2]
    if s.rotated:
        R = s.R
        x, y, z = (R[0, c] * x + R[1, c] * y + R[2, c] * z for c in range(3))
    L0, M0, N0 = out["L0"], out["M0"], out["N0"]
    w = out["w"]
    widx = O.wavelength_index(w, table.wavelengths)
    inten = out["i"]
    with np.errstate(all="ignore"):
        nx, ny, nz = PO._normal(s, x, y, [status])
        f = grating_vector(s, x, y, nx, ny, nz)
        L, M, N = grating_diffraction(s, L0, M0, N0, s.n1[widx], s.n2[widx], w, nx, ny, nz, *f)
        # coating step (interactions/base.py:111-128) with the unaligned normal
        if s.coating == T.COAT_SIMPLE:
            inten = inten * (s.coat_r if s.reflective else s.coat_t)
        elif s.coating == T.COAT_FRESNEL:
            if P is None:
                raise ValueError("Fresnel coating requires polarized rays")
            d = np.abs(nx * L0 + ny * M0 + nz * N0)
            J = O.fresnel_jones(np.arccos(np.clip(d, -1, 1)), s.coat_n1[widx], s.coat_n2[widx], s.reflective, x.size)
            P = O.polarized_update(P, L0, M0, N0, L, M, N, J)
        elif P is not None:
            P = O.polarized_update(P, L0, M0, N0, L, M, N, None)
        if s.rotated:
            R = s.R
            x, y, z = (R[r, 0] * x + R[r, 1] * y + R[r, 2] * z for r in range(3))
            L, M, N = (R[r, 0] * L + R[r, 1] * M + R[r, 2] * N for r in range(3))
        x, y, z = x + s.t[0], y + s.t[1], z + s.t[2]
    new = dict(x=x, y=y, z=z, L=L, M=M, N=N, i=inten, w=w, opd=out["opd"], L0=L0, M0=M0, N0=N0)
    return new, status, P


def trace(table: T.SurfaceTable, rays: dict, first: int = 0, last: int | None = None, polarized: bool = False):
    """``trace_oracle.trace`` for tables that may hold ruled gratings and phase-profile surfaces."""
    last = table.num_surfaces if last is None else last
    state = {k: np.asarray(v) for k, v in rays.items()}
    state.setdefault("opd", np.zeros_like(state["x"]))
    P = None
    if polarized:
        P = np.array(rays["p"]) if "p" in rays else np.tile(np.eye(3), (state["x"].size, 1, 1))
    rec = {k: [] for k in O.RECORD_KEYS}
    status = 0
    si = first
    out = None
    while si < last:
        if table.surfaces[si].interaction != T.INTERACT_GRATING:
            sj = si
            while sj < last and table.surfaces[sj].interaction != T.INTERACT_GRATING:
                sj += 1
            inp = dict(state)
            if polarized:
                inp["p"] = P
            out, r, st = PO.trace(table, inp, si, sj, polarized=polarized)
            if polarized:
                P = out["p"]
            for k in O.RECORD_KEYS:
                rec[k].extend(list(r[k]))
            si = sj
        else:
            out, st, P = _grating_surface(table, si, {k: v for k, v in state.items() if k != "p"}, P)
            vals = (out["x"], out["y"], out["z"], out["L"], out["M"], out["N"], out["i"], out["opd"])
            for k, v in zip(O.RECORD_KEYS, vals):
                rec[k].append(v.copy() if table.surfaces[si].record else np.full_like(v, np.nan))
            si += 1
        status |= st
        state = {k: out[k] for k in ("x", "y", "z", "L", "M", "N", "i", "w", "opd")}
    res = dict(state)
    res.update(L0=out["L0"] if out else None, M0=out["M0"] if out else None, N0=out["N0"] if out else None)
    if P is not None:
        res["p"] = P
    n = state["x"].size
    return res, {k: (np.stack(v) if v else np.zeros((0, n))) for k, v in rec.items()}, status
