"""TEST INFRASTRUCTURE ONLY -- the device-math stand-in for optiland_b200.plugin.CudaEngine (oracle/devmath_engine.py)
with the irradiance binning as well: ``irradiance`` runs the kernel's per-ray arithmetic compiled for the host
(oracle/hostcheck_irradiance.py), so that the plugin's ``IncoherentIrradiance`` wrapper runs live on a CPU."""
from oracle.devmath_engine import DeviceMathEngine


class IrradianceDeviceMathEngine(DeviceMathEngine):
    """TEST-ONLY: ``CudaEngine.irradiance``'s contract on host tensors."""

    def irradiance(self, x, y, z, power, x_edges, y_edges, frame):
        import torch

        from oracle.hostcheck_irradiance import bin_rays

        ts = (x, y, z, power)
        if not all(torch.is_tensor(t) and not t.is_cuda and t.dtype == x.dtype and t.ndim == 1 and t.shape == x.shape
                   and t.dtype in (torch.float32, torch.float64) for t in ts):
            return None
        self.calls.append(("irradiance", len(x_edges) - 1, len(y_edges) - 1, int(x.numel())))
        np_ = [t.detach().numpy() for t in ts]
        _, hist = bin_rays(np_[0], np_[1], np_[3], x_edges, y_edges, z=np_[2], frame=frame)
        return torch.from_numpy(hist)
