"""Cost of the ray gradients of the fused training step: bench.py --mode train's workload (8192 rays, the 300k-point / 2.02 M-tetrahedra
mesh, the tetra_nerf configuration, the model's initial field), one TetrahedraNerf training forward + loss + backward per step, with the
ray origins and directions plain tensors or requiring grad (what a camera optimizer upstream of the rays makes them), alternating.  Prints
one JSON line per mode (default / deterministic): median step time of each (CUDA events, after warm-up), the extra device memory of the
backward with ray gradients, the card and its power limit.  Needs a GPU."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
for p in (str(ROOT), str(ROOT / "tetra-nerf_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import oracle as orc  # noqa: E402
from tetranerf.b200 import synthetic as syn  # noqa: E402
from tetranerf.nerfstudio import model as tnm  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=8192)
    ap.add_argument("--points", type=int, default=300_000)
    ap.add_argument("--iters", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ray_grads_bench needs a GPU")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    V, C = syn.delaunay_mesh(a.points, seed=0)
    field = syn.random_field(len(V), 64, seed=3, kind="init")
    cfg = tnm.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), num_samples=128, num_fine_samples=128,
                                   use_biased_sampler=True)
    m = tnm.TetrahedraNerf(cfg)
    sd = {"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(C), "tetrahedra_field": torch.from_numpy(field)}
    sd.update(orc.init_mlp_params(0))
    m.load_state_dict(sd, strict=False)
    m = m.to(dev).train()
    o, d = (torch.from_numpy(x).to(dev) for x in syn.camera_rays(a.rays, seed=5000))
    target = torch.rand((a.rays, 3), generator=torch.Generator().manual_seed(9)).to(dev)

    def step(rays_grad: bool):
        oo, dd = (o.clone().requires_grad_(True), d.clone().requires_grad_(True)) if rays_grad else (o, d)
        out = m(tnm.RayBundle(origins=oo, directions=dd))
        m.get_loss_dict(out, {"image": target})["rgb_loss"].backward()
        if rays_grad:
            assert oo.grad is not None and dd.grad is not None
        m.zero_grad(set_to_none=True)

    for det in (False, True):
        os.environ["TETRANERF_B200_DETERMINISTIC"] = "1" if det else "0"
        torch.manual_seed(0)
        step(False)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info(dev)[0]
        step(True)
        torch.cuda.synchronize()
        extra = free0 - torch.cuda.mem_get_info(dev)[0]  # the tracer's dX rows (default mode) and per-sample dL/dx
        times = {False: [], True: []}
        for it in range(a.warmup + a.iters):
            for rg in (False, True):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                step(rg)
                e1.record()
                e1.synchronize()
                if it >= a.warmup:
                    times[rg].append(e0.elapsed_time(e1))
        plain, rays = float(np.median(times[False])), float(np.median(times[True]))
        print(json.dumps({"mode": "deterministic" if det else "default", "rays": a.rays, "tetrahedra": len(C), "iters": a.iters,
                          "step_ms": round(plain, 3), "step_ms_with_ray_grads": round(rays, 3), "extra_ms": round(rays - plain, 3),
                          "step_ms_range": [round(min(times[False]), 3), round(max(times[False]), 3)],
                          "step_ms_with_ray_grads_range": [round(min(times[True]), 3), round(max(times[True]), 3)],
                          "extra_device_bytes": int(extra), "gpu": q}), flush=True)


if __name__ == "__main__":
    main()
