"""Batched many-systems trace timing (SURVEY.md 8f-4): B perturbed Cooke triplets x m rays each, the
tolerancing Monte-Carlo shape (optiland/tolerancing/monte_carlo.py: one small trace per sampled system).

Arms, all on one GPU, CUDA-event timed:
  batch_records   one batched-table launch, shared launch rays, all record rows written
  batch_moments   one launch, shared launch rays, per-system spot moments only (no per-ray output)
  loop_single     B olb_trace launches on B pre-uploaded single-system tables (what a caller could do
                  without the batch entry point; table preparation NOT timed, so this is its best case)
Prints one JSON line per (B, m)."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from optiland_b200 import _lib  # noqa: E402
from optiland_b200.batch import BatchedTable, system_table, template_params, trace_batch  # noqa: E402
from optiland_b200.table import SurfaceTable  # noqa: E402
from optiland_b200.trace import DeviceTable, RealRays, trace_device  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def timed(fn, warm=3, reps=10):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    z = np.load(os.path.join(GOLDEN, "cooke_c1.npz"), allow_pickle=False)
    table = SurfaceTable.from_arrays(z)
    S = table.num_surfaces
    rays_np = {k: z["in_" + k] for k in ("x", "y", "z", "L", "M", "N", "i", "w")}
    dtype = torch.float32
    for B, m in ((1024, 1024), (4096, 1024), (16384, 256), (256, 65536)):
        rng = np.random.default_rng(0)
        p0 = template_params(table)
        P = np.repeat(p0[None], B, axis=0)
        P[:, 1:S - 1, _lib.BP_TX:_lib.BP_TX + 2] += rng.normal(0, 0.02, (B, S - 2, 2))
        P[:, 1:S - 1, _lib.BP_CURV] *= 1 + rng.normal(0, 1e-3, (B, S - 2))
        idx = rng.integers(0, rays_np["x"].size, size=m)
        one = {k: v[idx] for k, v in rays_np.items()}
        rays = RealRays(one["x"], one["y"], one["z"], one["L"], one["M"], one["N"], one["i"], one["w"], dtype=dtype)
        bt = BatchedTable(table, P)
        t_rec = timed(lambda: trace_batch(bt, rays, m, shared_input=True))
        t_mom = timed(lambda: trace_batch(bt, rays, m, shared_input=True, record=False, moments=True))
        nloop = min(B, 256)
        singles = [DeviceTable(system_table(table, P[b])) for b in range(nloop)]

        def loop():
            for d in singles:
                r = RealRays.__new__(RealRays)
                r.__dict__.update(rays.__dict__)
                trace_device(d, r, 0, S)

        t_loop = timed(loop, warm=1, reps=3) * (B / nloop)
        rs = B * m * S
        print(json.dumps({
            "workload": f"cooke triplet x {B} perturbed systems x {m} rays, fp32, shared launch rays",
            "batch_records_ms": round(t_rec, 4), "batch_records_ray_surfaces_per_s": rs / t_rec * 1e3,
            "batch_records_GBps": B * m * S * 32 / t_rec / 1e6,
            "batch_moments_ms": round(t_mom, 4), "batch_moments_ray_surfaces_per_s": rs / t_mom * 1e3,
            "loop_single_ms": round(t_loop, 3), "loop_measured_systems": nloop,
            "speedup_records_vs_loop": t_loop / t_rec, "speedup_moments_vs_loop": t_loop / t_mom}))


if __name__ == "__main__":
    main()
