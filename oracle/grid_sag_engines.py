"""TEST INFRASTRUCTURE ONLY -- a stand-in for optiland_b200.plugin.CudaEngine on boxes without a GPU that also traces
grid-sag surfaces (Optiland's ``GridSagGeometry``): the call shapes of ``oracle/phase_engines._PhaseEngine`` (trace,
fused pupil launch, spot moments, wavefront) with the trace done by the DEVICE ARITHMETIC compiled for the host with the
kernel variants the launcher picks for such tables (``oracle/hostcheck_grid_sag.py``,
tests/hostcheck/hostcheck_grid_sag.cpp).  Phase-profile, grating and coated tables take the same dispatch."""
from oracle.phase_engines import PhaseDeviceMathEngine


class GridSagDeviceMathEngine(PhaseDeviceMathEngine):
    """TEST-ONLY: the kernel's own arithmetic on the CPU, grid-sag surfaces included."""

    def _core(self, table, inp, first, last, pmat):
        import numpy as np

        from oracle.hostcheck_grid_sag import run_hostcheck_grid_sag

        return run_hostcheck_grid_sag(table, inp, np.float64, first, last, pmat=pmat)

    def trace_grad(self, table, params, rays, coefs=None):
        """TEST-ONLY differentiable engine: the host instantiation of the forward kernel and of the adjoint (its
        general variant, hostcheck.cpp's olbhc_backward_tables_*) -- the arithmetic of olb_trace_bwd_* without a GPU."""
        import ctypes as C

        import numpy as np
        import torch

        from oracle.hostcheck_api import load, run_backward
        from oracle.hostcheck_grid_sag import run_hostcheck_grid_sag
        from optiland_b200 import _lib
        from optiland_b200 import autograd as AG

        hc = load()
        ht = _lib.HostTable(table)
        if coefs is not None or not hc.olbhc_bwd_supported(C.byref(ht.c)):
            return None
        self.calls.append(("grad", table.num_surfaces, int(rays.x.numel())))
        keys = ("x", "y", "z", "L", "M", "N", "i", "opd")
        recs = ("x", "y", "z", "L", "M", "N", "intensity", "opd")

        class Fn(torch.autograd.Function):
            @staticmethod
            def forward(ctx, params, *ins):
                ctx.set_materialize_grads(False)
                tab = AG.params_to_table(table, params)
                inp = {k: t.detach().double().numpy() for k, t in zip(keys, ins)}
                inp["w"] = rays.w.detach().double().numpy()
                _, rec, _ = run_hostcheck_grid_sag(tab, inp, np.float64)
                ctx.tab, ctx.inp, ctx.rec = tab, inp, rec
                return tuple(torch.from_numpy(rec[k]) for k in recs)

            @staticmethod
            def backward(ctx, *grads):
                grec = {k: (None if g is None else g.double().numpy()) for k, g in zip(recs, grads)}
                gin, gpar, _ = run_backward(hc, ctx.tab, ctx.inp, ctx.rec, grec, tables=True)
                return (torch.from_numpy(gpar), *[torch.from_numpy(gin[k]) for k in keys])

        outs = Fn.apply(params, *[getattr(rays, k) for k in keys])
        rec = dict(zip(recs, outs))
        for k, key in zip(keys, recs):
            setattr(rays, k, rec[key][-1])
        return rec
