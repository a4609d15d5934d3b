"""Cost of the deterministic mode on the training benchmark workload (bench.py --mode train: 8192 rays, ~2.0 M-tetrahedra mesh,
tetra-nerf config): one training step (TetrahedraNerf.forward -> MSE loss -> backward -> RAdam step), every step from the same initial
state, in the default mode and under torch.use_deterministic_algorithms(True), alternating.  Prints per mode the median step time,
the backward kernel times of the last step, and the device memory the mode needs beyond the default: library workspace (cudaMalloc,
from cudaMemGetInfo) and the peak of torch's allocator.  Also checks that two deterministic steps give bitwise-equal gradients.

    python tools/determinism_bench.py [--steps 10] [--rays 8192] [--points 300000]
"""
import argparse
import os
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "tetra-nerf_b200")]
os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")  # torch's own matmuls under use_deterministic_algorithms (RAdam has none on the fused path)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed steps per mode and round")
    ap.add_argument("--rounds", type=int, default=2, help="alternating rounds (default, deterministic, default, ...)")
    ap.add_argument("--rays", type=int, default=8192)
    ap.add_argument("--points", type=int, default=bench.NUM_POINTS_TRAIN)
    args = ap.parse_args()
    os.environ.pop("TETRANERF_B200_DETERMINISTIC", None)
    os.environ["TETRANERF_B200_UNFUSED_TRAIN"] = "0"
    from tetranerf.nerfstudio import model as tnm

    dev = torch.device("cuda:0")
    syn = bench.synthetic()
    V, C = syn.delaunay_mesh(args.points, seed=0)
    field = syn.random_field(len(V), 64, seed=3, kind="init")
    w = bench.WORKLOADS["tetra-nerf"]
    cfg = tnm.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), num_samples=w["num_samples"],
                                   num_fine_samples=w["num_fine_samples"], use_biased_sampler=w["use_biased_sampler"])
    model = tnm.TetrahedraNerf(cfg)
    sd = {"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(C), "tetrahedra_field": torch.from_numpy(field)}
    sd.update(bench.mlp_params())
    model.load_state_dict(sd, strict=False)
    model = model.to(dev).train()
    opt = torch.optim.RAdam(model.parameters(), lr=1e-3)
    init = [p.detach().clone() for p in model.parameters()]
    R = args.rays
    o, d = syn.camera_rays(R, seed=5000)
    o, d = torch.from_numpy(o).to(dev), torch.from_numpy(d).to(dev)
    tgt = torch.from_numpy(np.random.default_rng(9000).random((R, 3), dtype=np.float32)).to(dev)

    def step():
        with torch.no_grad():
            for p, p0 in zip(model.parameters(), init):
                p.copy_(p0)
        opt.state.clear()
        torch.manual_seed(0)  # the stratified draws
        out = model(tnm.RayBundle(origins=o, directions=d))
        loss = model.get_loss_dict(out, {"image": tgt})["rgb_loss"]
        opt.zero_grad(set_to_none=True)
        loss.backward()
        grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
        opt.step()
        return grads

    def used():
        torch.cuda.synchronize(dev)
        torch.cuda.empty_cache()
        free, total = torch.cuda.mem_get_info(dev)
        return total - free

    res = {False: {"ms": [], "peak": 0}, True: {"ms": [], "peak": 0}}
    mem = {}
    fr = None
    for rnd in range(args.rounds):
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            step()  # warm-up (allocates the mode's workspace)
            if fr is None:
                fr = model._fused
                fr.set_profiling(True)
            mem.setdefault(det, used())
            torch.cuda.reset_peak_memory_stats(dev)
            for _ in range(args.steps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                step()
                b.record()
                torch.cuda.synchronize(dev)
                res[det]["ms"].append(a.elapsed_time(b))
            res[det]["peak"] = max(res[det]["peak"], torch.cuda.max_memory_allocated(dev))
            res[det]["bwd"] = fr.backward_timings_ms()
    torch.use_deterministic_algorithms(True)
    g1, g2 = step(), step()
    repeatable = all(torch.equal(g1[n], g2[n]) for n in g1)
    torch.use_deterministic_algorithms(False)

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"GPU: {torch.cuda.get_device_name(dev)}; power limit: {q.stdout.strip().split(',')[-1].strip() if q.returncode == 0 else 'unknown'}")
    print(f"workload: {R} rays, {len(C)} tetrahedra, tetra-nerf config; {args.rounds} x {args.steps} timed steps per mode, alternating")
    for det in (False, True):
        ms = res[det]["ms"]
        bw = ", ".join(f"{k} {v:.2f}" for k, v in res[det]["bwd"].items())
        print(f"{'deterministic' if det else 'default      '}: step median {statistics.median(ms):.2f} ms (min {min(ms):.2f}, max {max(ms):.2f}); "
              f"backward kernels (ms): {bw}; torch peak {res[det]['peak'] / 2**20:.0f} MiB")
    extra_lib = mem[True] - mem[False]
    extra_torch = res[True]["peak"] - res[False]["peak"]
    print(f"deterministic mode: +{statistics.median(res[True]['ms']) - statistics.median(res[False]['ms']):.2f} ms per step; "
          f"extra device memory: library workspace {extra_lib / 2**20:.0f} MiB, torch allocator peak {extra_torch / 2**20:+.0f} MiB")
    print(f"two deterministic steps bitwise equal: {repeatable}")


if __name__ == "__main__":
    main()
