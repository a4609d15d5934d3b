"""Cost and gain of occupancy sampling (DESIGN §4.13) against culling only (§4.12) on the fused paths.  Scene: synthetic.surface_scene
(two opaque spheres, k = 100, in otherwise empty space) on Delaunay meshes of 45k and 300k points (~0.30 M and ~2.02 M tetrahedra),
tetra_nerf settings (biased sampler) at 128 + 128, 64 + 64 and 32 + 32 samples, threshold 0.01.  Per mesh and sample count it prints one
JSON line with, for culling only and for placement: the mean |rgb - reference| over 4096 rays, the reference being the culled single
pass at 4096 samples (with its own distance to the 2048-sample pass, to show it has converged); the live (not culled) fraction of the
coarse and fine samples; the eval render's median time (4096 rays, f16w2); the training step's (8192 rays, saved forward + backward,
default mode), the two variants alternating run by run.  Times are CUDA events.  Every line carries the card, its power limit and
clocks, read in the same run.  Needs a GPU."""
from __future__ import annotations

import argparse
import ctypes
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
from tetranerf.b200 import synthetic as syn  # noqa: E402
from occupancy_bench import _timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, nargs="+", default=[45000, 300000])
    ap.add_argument("--samples", type=int, nargs="+", default=[128, 64, 32])
    ap.add_argument("--threshold", type=float, default=0.01)
    ap.add_argument("--iters", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("occupancy_sampling_bench needs a GPU")
    from tetranerf import cpp
    from tetranerf.b200.render import FusedRenderer, RenderSettings

    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    cudart = ctypes.CDLL("libcudart.so")

    def grab(ptr, shape):
        t = torch.empty(shape, dtype=torch.int32, device=dev)
        cudart.cudaMemcpy(ctypes.c_void_p(t.data_ptr()), ctypes.c_void_p(ptr), ctypes.c_size_t(t.numel() * 4), ctypes.c_int(3))
        return t

    for n in a.points:
        V, C = syn.delaunay_mesh(n, seed=0)
        field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
        tr = cpp.TetrahedraTracer(dev)
        tr.load_tetrahedra(torch.from_numpy(V).to(dev), torch.from_numpy(C).to(dev))
        fr = FusedRenderer(tr)
        fr.set_field(torch.from_numpy(field).to(dev))
        fr.set_weights(params)
        occ = torch.zeros(len(C), dtype=torch.float32, device=dev)
        fr.update_occupancy(occ, 0.0)
        o4, d4 = (torch.from_numpy(x).to(dev) for x in syn.camera_rays(4096, seed=5000))
        o8, d8 = (torch.from_numpy(x).to(dev) for x in syn.camera_rays(8192, seed=5001))
        fr.set_mlp_precision(2)
        fr.set_occupancy(occ, a.threshold)
        dense = lambda s: fr.render(o4, d4, RenderSettings(512, s, 0, True, 6.0))["rgb"].clone()  # noqa: E731
        ref = dense(4096)
        converged = (dense(2048) - ref).abs().mean().item()
        for S in a.samples:
            st = RenderSettings(512, S, S, True, 6.0)
            S2 = 2 * S + 1
            res = {"case": "occupancy_sampling", "points": n, "tetrahedra": len(C), "samples": f"{S}+{S}", "threshold": a.threshold,
                   "ref_2048_vs_4096": round(converged, 6)}
            g = torch.Generator(device="cpu").manual_seed(1)
            jc = torch.rand((8192, S + 1), generator=g).to(dev)
            jf = torch.rand((8192, S + 1), generator=g).to(dev)
            g_rgb = (torch.randn((8192, 3), generator=g) * 1e-3).to(dev)
            for place, nm in ((False, "cull"), (True, "place")):
                fr.set_occupancy(occ, a.threshold, place_samples=place)
                rgb = fr.render(o4, d4, st)["rgb"]
                res[f"err_{nm}"] = round((rgb - ref).abs().mean().item(), 6)
                bufs = fr.debug_buffers()
                na = int(grab(bufs["n_active"], (1,))[0])
                for key, SS, pn in (("vi_c", S, "coarse"), ("vi_f", S2, "fine")):
                    v = grab(bufs[key], (na, SS, 4))
                    res[f"live_{pn}_{nm}"] = round(1.0 - ((v[..., 0] == -1) & (v[..., 3] == -2)).float().mean().item(), 4)
            tr_ms, tt_ms = {False: [], True: []}, {False: [], True: []}
            for i in range(a.warmup + a.iters):
                for place in (False, True):
                    fr.set_occupancy(occ, a.threshold, place_samples=place)
                    t = _timed(lambda: fr.render(o4, d4, st), 1, 0)[0]

                    def step():
                        _, state = fr.train_forward_saved(o8, d8, st, jc, jf)
                        fr.train_backward_saved(state, g_rgb, None, len(V))

                    u = _timed(step, 1, 0)[0]
                    if i >= a.warmup:
                        tr_ms[place].append(t)
                        tt_ms[place].append(u)
            for place, nm in ((False, "cull"), (True, "place")):
                res[f"render_ms_f16w2_{nm}"] = round(float(np.median(tr_ms[place])), 3)
                res[f"train_ms_{nm}"] = round(float(np.median(tt_ms[place])), 3)
            res["gpu"] = gpu
            print(json.dumps(res), flush=True)
        fr.set_occupancy(None)


if __name__ == "__main__":
    main()
