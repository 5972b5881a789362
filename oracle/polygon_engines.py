"""TEST INFRASTRUCTURE ONLY -- a stand-in for optiland_b200.plugin.CudaEngine on boxes without a GPU that also traces
tables with polygon apertures (Optiland's ``PolygonAperture`` / ``FileAperture``): ``GridSagDeviceMathEngine`` with the
trace done by the kernel variants the launcher picks for such tables (``oracle/hostcheck_polygon.py``,
tests/hostcheck/hostcheck_polygon.cpp).  Every other table takes the same dispatch as before."""
from oracle.grid_sag_engines import GridSagDeviceMathEngine


class PolygonDeviceMathEngine(GridSagDeviceMathEngine):
    """TEST-ONLY: the kernel's own arithmetic on the CPU, polygon apertures included."""

    def _core(self, table, inp, first, last, pmat):
        import numpy as np

        from oracle.hostcheck_polygon import run_hostcheck_polygon

        return run_hostcheck_polygon(table, inp, np.float64, first, last, pmat=pmat)

    def trace_grad(self, table, params, rays, coefs=None):
        """The parent's differentiable engine with the forward pass through the polygon-aware dispatch (the adjoint is
        hostcheck.cpp's general variant, which holds the polygon scan)."""
        from unittest import mock

        from oracle.hostcheck_polygon import run_hostcheck_polygon

        with mock.patch("oracle.hostcheck_grid_sag.run_hostcheck_grid_sag", run_hostcheck_polygon):
            return super().trace_grad(table, params, rays, coefs)
