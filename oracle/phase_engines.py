"""TEST INFRASTRUCTURE ONLY -- stand-ins for optiland_b200.plugin.CudaEngine on boxes without a GPU that also trace
phase-profile surfaces (``PhaseInteractionModel``): the same call shapes as ``OracleEngine`` / ``DeviceMathEngine``
(trace, fused pupil launch, spot moments, wavefront), with the trace itself done by

``PhaseOracleEngine``      the NumPy restatement (``oracle/phase_oracle.py`` on top of ``oracle/trace_oracle.py``);
``PhaseDeviceMathEngine``  the DEVICE ARITHMETIC compiled for the host with the kernel variants the launcher picks for
                           phase tables (``oracle/hostcheck_phase.py``, tests/hostcheck/hostcheck_phase.cpp).

PSF, FFT-PSF and the adjoint are inherited from ``OracleEngine`` (the plugin never asks for an adjoint of a phase
table: it declines such gradients first)."""
import numpy as np

from oracle.oracle_engine import OracleEngine, raise_status

_KEYS = ("x", "y", "z", "L", "M", "N", "i", "w", "opd")


class _PhaseEngine(OracleEngine):
    """The call shapes over one trace core ``_core(table, inp, first, last, pmat) -> (out, rec, status)`` (fp64 numpy;
    ``pmat``: (n, 3, 3) complex P matrices or None)."""

    def _core(self, table, inp, first, last, pmat):
        raise NotImplementedError

    def _pol_intensity(self, P, k0, i0, state):
        raise NotImplementedError

    def _wavefront(self, fin, px, py, ref):
        raise NotImplementedError

    def trace(self, table, rays, first, last):
        import torch

        self.calls.append((table.num_surfaces, int(rays.x.numel())))
        n = int(rays.x.numel())
        inp = {k: np.broadcast_to(getattr(rays, k).detach().double().numpy(), (n,)).copy() for k in _KEYS}
        polarized = type(rays).__name__ == "PolarizedRays"
        pmat = rays.p.detach().numpy().astype(np.complex128) if polarized else None
        out, rec, status = self._core(table, inp, first, last, pmat)
        raise_status(status)
        if polarized:
            rays.p = torch.from_numpy(out["p"])
        dt = rays.x.dtype
        for k in ("x", "y", "z", "L", "M", "N", "i", "opd"):
            setattr(rays, k, torch.from_numpy(np.asarray(out[k])).to(dt))
        return {k: torch.from_numpy(v).to(dt) for k, v in rec.items()}

    def _launch(self, table, Px, Py, affine, wavelength=None):
        from optiland_b200.launch import launch_from_affine

        px, py = Px.detach().double().numpy(), Py.detach().double().numpy()
        aff = dict(affine)
        if aff.get("fields") is not None:
            aff["fields"] = tuple(t.detach().double().numpy() for t in aff["fields"])
        x, y, z, L, M, N = launch_from_affine(px, py, aff)
        w = wavelength.detach().double().numpy() if wavelength is not None else np.full_like(px, table.wavelengths[0])
        return px, py, dict(x=x, y=y, z=z, L=L, M=M, N=N, i=np.full_like(px, affine.get("intensity", 1.0)), w=w)

    def trace_pupil(self, table, Px, Py, affine, wavelength=None, polarization=False):
        import torch

        self.calls.append(("pupil", table.num_surfaces, int(Px.numel())))
        px, py, inp = self._launch(table, Px, Py, affine, wavelength)
        pmat = None if polarization is False else np.tile(np.eye(3, dtype=np.complex128), (px.size, 1, 1))
        out, rec, status = self._core(table, inp, 0, table.num_surfaces, pmat)
        raise_status(status)
        res = {k: torch.from_numpy(v).to(Px.dtype) for k, v in rec.items()}
        if polarization is False:
            return res
        res["p"] = torch.from_numpy(out["p"]).to(torch.complex128 if Px.dtype == torch.float64 else torch.complex64)
        if polarization == "matrix":
            res["i_pol"] = res["intensity"][-1]
        else:
            k0 = (inp["L"], inp["M"], inp["N"])
            res["i_pol"] = torch.from_numpy(self._pol_intensity(out["p"], k0, inp["i"], polarization)).to(Px.dtype)
        return res

    def spot_moments(self, table, Px, Py, affine, center=(0.0, 0.0), last=None, global_xy=False, every_ray=False):
        self.calls.append(("moments", table.num_surfaces, int(Px.numel())))
        _, _, inp = self._launch(table, Px, Py, affine)
        last = table.num_surfaces if last is None else last
        _, rec, status = self._core(table, inp, 0, last, None)
        raise_status(status)
        gx, gy, ii, oo = rec["x"][-1], rec["y"][-1], rec["intensity"][-1], rec["opd"][-1]
        if not global_xy:
            s = table.surfaces[last - 1]
            loc = np.asarray(s.R).T @ np.stack([gx - s.t[0], gy - s.t[1], rec["z"][-1] - s.t[2]])
            gx, gy = loc[0], loc[1]
        dx, dy = gx - center[0], gy - center[1]
        fin_ok = np.isfinite(dx) & np.isfinite(dy)
        keep = np.ones_like(fin_ok) if every_ray else ((ii > 0) & fin_ok)
        return [float(keep.sum()), float(dx[keep].sum()), float(dy[keep].sum()), float((dx[keep] ** 2 + dy[keep] ** 2).sum()),
                float(ii[keep].sum()), float(oo[keep].sum()), float((oo[keep] ** 2).sum()),
                0.0 if every_ray else float(((ii > 0) & ~fin_ok).sum())]

    def trace_wavefront(self, table, Px, Py, affine, ref, polarized=False):
        import torch

        self.calls.append(("wavefront", table.num_surfaces, int(Px.numel())))
        px, py, inp = self._launch(table, Px, Py, affine)
        pmat = np.tile(np.eye(3, dtype=np.complex128), (px.size, 1, 1)) if polarized else None
        fin, _, status = self._core(table, inp, 0, table.num_surfaces, pmat)
        raise_status(status)
        out = self._wavefront(fin, px, py, ref)
        res = {k: torch.from_numpy(np.asarray(v)).to(Px.dtype) for k, v in out.items()}
        if polarized:
            res["p"] = torch.from_numpy(fin["p"]).to(torch.complex128 if Px.dtype == torch.float64 else torch.complex64)
        return res


class PhaseOracleEngine(_PhaseEngine):
    """TEST-ONLY: the NumPy restatement of the reference, phase-profile surfaces included."""

    def _core(self, table, inp, first, last, pmat):
        from oracle import phase_oracle

        if pmat is not None:
            inp = dict(inp, p=pmat)
        return phase_oracle.trace(table, inp, first, last, polarized=pmat is not None)

    def _pol_intensity(self, P, k0, i0, state):
        from oracle import trace_oracle as O

        return O.polarized_intensity(P, *k0, i0, state)

    def _wavefront(self, fin, px, py, ref):
        from oracle import trace_oracle as O

        return O.wavefront_reference_sphere(fin, px, py, ref)


class PhaseDeviceMathEngine(_PhaseEngine):
    """TEST-ONLY: the kernel's own arithmetic on the CPU, phase-profile surfaces included."""

    def _core(self, table, inp, first, last, pmat):
        from oracle.hostcheck_phase import run_hostcheck_phase

        return run_hostcheck_phase(table, inp, np.float64, first, last, pmat=pmat)

    def _pol_intensity(self, P, k0, i0, state):
        from oracle.hostcheck_api import load, run_pol_intensity
        from optiland_b200 import table as T

        out, st = run_pol_intensity(load(), P, k0, i0, state)
        if st & T.ST_K_PARALLEL_X:
            raise ValueError("k-vector parallel to x-axis is not currently supported.")
        return out

    def _wavefront(self, fin, px, py, ref):
        from oracle.hostcheck_api import load, run_wavefront

        out = run_wavefront(load(), fin, px, py, ref)
        out["intensity"] = fin["i"]
        return out
