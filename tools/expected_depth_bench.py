"""Cost of the expected depth (DESIGN §4.10) on bench.py's workload (the 45k-point / 302k-tetrahedra mesh, torch-default network on the
"normal" field): alternating renders with and without it (4096 rays; tetra_nerf and tetra_nerf_original, both MLP precisions), and
alternating 8192-ray training steps (forward + backward, tetra_nerf, GradientScaler) with a loss on rgb and with a loss on rgb + the
expected depth, in the default and the deterministic mode.  Prints one JSON line per case: median call time of each (CUDA events,
after warm-up), the card, its power limit and clocks.  Needs a GPU."""
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


def _alternate(fns, warmup, iters):
    times = [[] for _ in fns]
    for it in range(warmup + iters):
        for k, fn in enumerate(fns):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            if it >= warmup:
                times[k].append(e0.elapsed_time(e1))
    return [float(np.median(t)) for t in times]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=4096)
    ap.add_argument("--train-rays", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("expected_depth_bench needs a GPU")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    V, C = syn.delaunay_mesh(45000, seed=0)
    tr = cpp.TetrahedraTracer(dev)
    tr.load_tetrahedra(torch.from_numpy(V).to(dev), torch.from_numpy(C).to(dev))
    fr = FusedRenderer(tr)
    fr.set_field(torch.from_numpy(syn.random_field(len(V), 64, seed=3)).to(dev))
    fr.set_weights(orc.init_mlp_params(0))
    o, d = syn.camera_rays(a.rays)
    o, d = torch.from_numpy(o).to(dev), torch.from_numpy(d).to(dev)
    for cfg in ("tetra_nerf", "tetra_nerf_original"):
        st = getattr(RenderSettings, cfg)()
        for prec, pname in ((2, "f16w2"), (3, "bf16x3")):
            fr.set_mlp_precision(prec)
            out = fr.render(o, d, st, expected_depth=True)
            plain, ed = _alternate([lambda: fr.render(o, d, st, out=out), lambda: fr.render(o, d, st, out=out, expected_depth=True)],
                                   a.warmup, a.iters)
            print(json.dumps({"case": "eval", "config": cfg, "mlp_precision": pname, "rays": a.rays, "plain_ms": round(plain, 4),
                              "expected_depth_ms": round(ed, 4), "extra_ms": round(ed - plain, 4), "gpu": q}), flush=True)
    R = a.train_rays
    o, d = syn.camera_rays(R, seed=2)
    o, d = torch.from_numpy(o).to(dev), torch.from_numpy(d).to(dev)
    st = RenderSettings.tetra_nerf()
    g = torch.Generator().manual_seed(0)
    jc = torch.rand((R, st.num_samples + 1), generator=g).to(dev)
    jf = torch.rand((R, st.num_fine_samples + 1), generator=g).to(dev)
    target = torch.rand((R, 3), generator=g).to(dev)

    def step(depth):
        out, state = fr.train_forward_saved(o, d, st, jc, jf, expected_depth=depth)
        g_rgb = (2.0 * (out["rgb"] - target) / (3 * R)).contiguous()
        g_ed = ((out["expected_depth"][:, 0] - 1.0) * (2.0 / R)).contiguous() if depth else None
        fr.train_backward_saved(state, g_rgb, None, len(V), True, grad_expected_depth=g_ed)

    for mode in ("default", "deterministic"):
        torch.use_deterministic_algorithms(mode == "deterministic")  # the fused step's mode follows it (FusedRenderer._train_args)
        plain, ed = _alternate([lambda: step(False), lambda: step(True)], a.warmup, a.iters)
        torch.use_deterministic_algorithms(False)
        print(json.dumps({"case": "train_step", "config": "tetra_nerf", "mode": mode, "rays": R, "rgb_loss_ms": round(plain, 4),
                          "rgb_depth_loss_ms": round(ed, 4), "extra_ms": round(ed - plain, 4), "gpu": q}), flush=True)


if __name__ == "__main__":
    main()
