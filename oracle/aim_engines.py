"""TEST INFRASTRUCTURE ONLY -- a stand-in for optiland_b200.plugin.CudaEngine on boxes without a GPU that also runs
the ray-aiming solve (``CudaEngine.aim``): ``DeviceMathEngine`` plus ``aim`` through the CPU instantiation of
olb_aim.cuh (``oracle/hostcheck_aim.py``).  With it the plugin's device robust aimer runs end to end on the CPU."""
import numpy as np

from oracle.devmath_engine import DeviceMathEngine


class AimDeviceMathEngine(DeviceMathEngine):
    """TEST-ONLY: ``DeviceMathEngine`` with ``aim``."""

    def aim(self, table, guess, Px, Py, r_stop, J_factor, tol, max_iter, infinite):
        import torch

        from oracle.hostcheck_aim import run_aim

        n = int(guess["x"].numel())
        self.calls.append(("aim", table.num_surfaces, n))
        g = {k: v.detach().double().numpy() for k, v in guess.items()}
        dt = np.float64 if guess["x"].dtype == torch.float64 else np.float32
        sol, status, _ = run_aim(table, g, Px.detach().double().numpy(), Py.detach().double().numpy(), 0,
                                 table.num_surfaces, r_stop, J_factor, tol, max_iter, infinite, dtype=dt)
        for k in ("x", "y", "L", "M"):
            guess[k].copy_(torch.from_numpy(sol[k]))
        return status
