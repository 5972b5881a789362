"""TEST INFRASTRUCTURE ONLY -- CPU restatement (NumPy, fp64) of Optiland's ``PhaseInteractionModel``
(optiland/interactions/phase_interaction_model.py:45-132) with the profiles of optiland/phase/{constant,
linear_grating,radial}.py, on top of the NumPy oracle of the trace loop (``oracle/trace_oracle.py``).

``trace`` has the signature and the results of ``trace_oracle.trace``.  Runs of refractive / reflective surfaces go
through ``trace_oracle.trace`` unchanged; a phase surface is traced there with its interaction and coating taken off
(localize, distance, propagation, OPD, absorption and aperture are the same for both models), and the phase
interaction, the coating step and the efficiency are applied here, in the surface's local frame.
"""
from __future__ import annotations

import dataclasses

import numpy as np

from oracle import trace_oracle as O
from optiland_b200 import table as T


def phase_interaction(s: T.SurfaceSpec, x, y, L, M, N, n1, n2, w, inten, opd, nx, ny, nz):
    """interact_real_rays up to the coating step, with the geometry's own (unaligned) normal.  Returns
    (L, M, N, intensity, opd)."""
    if s.reflective:
        n2 = n1
    k0 = 2 * np.pi / (w * 1e-3)
    c = s.phase_terms
    if s.interaction == T.INTERACT_PHASE_CONSTANT:
        phase, gx, gy = np.full_like(x, c[0]), np.zeros_like(x), np.zeros_like(x)
    elif s.interaction == T.INTERACT_PHASE_LINEAR:
        phase, gx, gy = c[0] * x + c[1] * y, np.full_like(x, c[0]), np.full_like(x, c[1])
    else:
        r2 = x**2 + y**2
        r = np.sqrt(r2)
        phase, dr = np.zeros_like(x), np.zeros_like(x)
        for i, a in enumerate(c):
            p = i + 1
            phase = phase + a * r2**p
            dr = dr + a * 2 * p * r ** (2 * p - 1)
        safe = np.where(r == 0, 1.0, r)
        gx = np.where(r == 0, 0.0, dr / safe * x)
        gy = np.where(r == 0, 0.0, dr / safe * y)
    gdn = gx * nx + gy * ny
    Gx, Gy, Gz = gx - gdn * nx, gy - gdn * ny, -gdn * nz
    kx, ky, kz = n1 * k0 * L, n1 * k0 * M, n1 * k0 * N
    kdn = kx * nx + ky * ny + kz * nz
    px, py, pz = kx - kdn * nx + Gx, ky - kdn * ny + Gy, kz - kdn * nz + Gz
    R2 = (n2 * k0) ** 2 - (px**2 + py**2 + pz**2)
    inten = np.where(R2 < 0.0, np.zeros_like(inten), inten)
    alpha = (-1.0 if s.reflective else 1.0) * np.sqrt(np.maximum(0.0, R2))
    ox, oy, oz = px + alpha * nx, py + alpha * ny, pz + alpha * nz
    mag = np.sqrt(ox**2 + oy**2 + oz**2)
    return ox / mag, oy / mag, oz / mag, inten, opd - phase / k0


def _normal(s: T.SurfaceSpec, x, y, status):
    if s.kind == T.GEOM_PLANE:
        return np.zeros_like(x), np.zeros_like(x), np.ones_like(x)
    if s.kind == T.GEOM_STANDARD:
        return O.conic_normal(x, y, s.radius, s.conic)
    return O._sag_and_normal_fns(s, status)[1](x, y)


def _phase_surface(table, si, state, P):
    """One phase surface: (state after it, its record row values, P, status)."""
    s = table.surfaces[si]
    bare = dataclasses.replace(s, interaction=T.INTERACT_REFRACT, coating=T.COAT_NONE, coat_n1=None, coat_n2=None,
                               record=True)
    surfaces = list(table.surfaces)
    surfaces[si] = bare
    out, _, status = O.trace(T.SurfaceTable(surfaces, table.wavelengths), state, si, si + 1)
    st = [status]
    # back into the local frame of the surface (the oracle hands back global coordinates)
    x, y, z = out["x"] - s.t[0], out["y"] - s.t[1], out["z"] - s.t[2]
    if s.rotated:
        R = s.R
        x, y, z = (R[0, c] * x + R[1, c] * y + R[2, c] * z for c in range(3))
    L0, M0, N0 = out["L0"], out["M0"], out["N0"]
    w = out["w"]
    widx = O.wavelength_index(w, table.wavelengths)
    with np.errstate(all="ignore"):
        nx, ny, nz = _normal(s, x, y, st)
        L, M, N, inten, opd = phase_interaction(s, x, y, L0, M0, N0, s.n1[widx], s.n2[widx], w, out["i"], out["opd"],
                                                nx, ny, nz)
        # coating step (interactions/base.py:111-128) with the same normal
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
        inten = inten * s.phase_efficiency
        if s.rotated:
            R = s.R
            x, y, z = (R[r, 0] * x + R[r, 1] * y + R[r, 2] * z for r in range(3))
            L, M, N = (R[r, 0] * L + R[r, 1] * M + R[r, 2] * N for r in range(3))
        x, y, z = x + s.t[0], y + s.t[1], z + s.t[2]
    new = dict(x=x, y=y, z=z, L=L, M=M, N=N, i=inten, w=w, opd=opd, L0=L0, M0=M0, N0=N0)
    return new, st[0], P


def trace(table: T.SurfaceTable, rays: dict, first: int = 0, last: int | None = None, polarized: bool = False):
    """``trace_oracle.trace`` for tables that may hold phase-profile surfaces."""
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
        if table.surfaces[si].interaction == T.INTERACT_REFRACT:
            sj = si
            while sj < last and table.surfaces[sj].interaction == T.INTERACT_REFRACT:
                sj += 1
            inp = dict(state)
            if polarized:
                inp["p"] = P
            out, r, st = O.trace(table, inp, si, sj, polarized=polarized)
            if polarized:
                P = out["p"]
            for k in O.RECORD_KEYS:
                rec[k].extend(list(r[k]))
            si = sj
        else:
            out, st, P = _phase_surface(table, si, {k: v for k, v in state.items() if k != "p"}, P)
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

