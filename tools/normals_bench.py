"""Cost of the normal map: alternating plain and normals renders of bench.py's workload (4096 rays, the 45k-point / 302k-tetrahedra
mesh, torch-default network on the "normal" field), in the tetra_nerf and tetra_nerf_original configurations and both MLP precisions.
Prints one JSON line per case: median call time of each (CUDA events, after warm-up), the extra device memory, the card and its power
limit.  Needs a GPU."""
from __future__ import annotations

import argparse
import json
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
from tetranerf import cpp  # noqa: E402
from tetranerf.b200 import synthetic as syn  # noqa: E402
from tetranerf.b200.render import FusedRenderer, RenderSettings  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("normals_bench needs a GPU")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    V, C = syn.delaunay_mesh(45000, seed=0)
    o, d = syn.camera_rays(a.rays)
    o, d = torch.from_numpy(o).to(dev), torch.from_numpy(d).to(dev)
    tr = cpp.TetrahedraTracer(dev)
    tr.load_tetrahedra(torch.from_numpy(V).to(dev), torch.from_numpy(C).to(dev))
    fr = FusedRenderer(tr)
    fr.set_field(torch.from_numpy(syn.random_field(len(V), 64, seed=3)).to(dev))
    fr.set_weights(orc.init_mlp_params(0))
    for cfg in ("tetra_nerf", "tetra_nerf_original"):
        st = getattr(RenderSettings, cfg)()
        for prec, pname in ((2, "f16w2"), (3, "bf16x3")):
            fr.set_mlp_precision(prec)
            out = fr.render(o, d, st)
            torch.cuda.synchronize()
            m0 = torch.cuda.mem_get_info(dev)[0]
            fr.render(o, d, st, out=out, normals=True)
            torch.cuda.synchronize()
            extra = m0 - torch.cuda.mem_get_info(dev)[0]  # tracer workspace + the [R,3] output
            times = {False: [], True: []}
            for it in range(a.warmup + a.iters):
                for nm in (False, True):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    fr.render(o, d, st, out=out, normals=nm)
                    e1.record()
                    e1.synchronize()
                    if it >= a.warmup:
                        times[nm].append(e0.elapsed_time(e1))
            plain, nrm = float(np.median(times[False])), float(np.median(times[True]))
            print(json.dumps({"config": cfg, "mlp_precision": pname, "rays": a.rays, "plain_ms": round(plain, 4), "normals_ms": round(nrm, 4),
                              "extra_ms": round(nrm - plain, 4), "extra_device_bytes": int(extra), "gpu": q}), flush=True)


if __name__ == "__main__":
    main()
