"""Time of the surface extraction (tn_surface_extract + tn_surface_copy through FusedRenderer.extract_surface) on the mesh of
bench.py --mode train (300k points, ~2.02 M tetrahedra) with synthetic.surface_scene at sharpness k = 1000 and level ln 2.  Prints the GPU's
name and power limit, the mesh and surface sizes, the median / min / max time of the timed calls (host clock around each call, which
ends in a device synchronise) and the library's workspace (cudaMemGetInfo before and after the first call).

    python tools/surface_bench.py [--points 300000] [--k 1000] [--reps 10] [--warmup 2]
"""
import argparse
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "tetra-nerf_b200")]

import numpy as np  # noqa: E402
import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=300_000)
    ap.add_argument("--k", type=float, default=1000.0)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    from oracle import oracle as orc
    from tetranerf import cpp
    from tetranerf.b200 import synthetic as syn
    from tetranerf.b200.render import FusedRenderer

    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"GPU: {torch.cuda.get_device_name(dev)}; power limit: {q.stdout.strip().split(',')[-1].strip() if q.returncode == 0 else 'unknown'}")
    V, C = syn.delaunay_mesh(args.points, seed=0)
    field, params = syn.surface_scene(V, args.k, orc.init_mlp_params(0))
    tr = cpp.TetrahedraTracer(dev)
    xyz, cells = torch.from_numpy(V).to(dev), torch.from_numpy(C).to(dev)
    tr.load_tetrahedra(xyz, cells)
    fr = FusedRenderer(tr)
    fr.set_field(torch.from_numpy(field).to(dev))
    fr.set_weights(params)
    torch.cuda.synchronize(dev)
    level = float(np.log(2.0))
    free0 = torch.cuda.mem_get_info(dev)[0]
    times = []
    for i in range(args.warmup + args.reps):
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        surf = fr.extract_surface(level)
        torch.cuda.synchronize(dev)
        if i == 0:
            workspace = free0 - torch.cuda.mem_get_info(dev)[0] - sum(t.numel() * t.element_size() for t in surf.values())
        if i >= args.warmup:
            times.append((time.perf_counter() - t0) * 1e3)
    n, f = surf["vertices"].shape[0], surf["faces"].shape[0]
    print(f"mesh: {len(V)} vertices, {len(C)} tetrahedra; surface (k = {args.k:g}, level ln 2): {n} vertices, {f} faces")
    print(f"extract_surface: median {statistics.median(times):.2f} ms (min {min(times):.2f}, max {max(times):.2f}) over {len(times)} calls; "
          f"library workspace ~{workspace / 2**20:.0f} MiB (cudaMemGetInfo, includes allocator rounding)")


if __name__ == "__main__":
    main()
