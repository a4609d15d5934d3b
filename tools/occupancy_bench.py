"""Cost and gain of occupancy culling (DESIGN §4.12) on the fused paths.  Scene: synthetic.surface_scene (two opaque spheres, k = 100, in
otherwise empty space) on Delaunay meshes of 45k and 300k points (~0.30 M and ~2.02 M tetrahedra), tetra_nerf settings, threshold 0.01.
Per mesh it prints one JSON line with: the culled fraction of the coarse and fine passes of the eval render; the eval render's median time
(4096 rays, f16w2 and bf16x3) and the training step's (8192 rays, saved forward + backward, default mode) with and without culling,
alternating run by run; and tn_occupancy_update's median time.  Times are CUDA events.  Every line carries the card, its power limit
and clocks, read in the same run.  Needs a GPU."""
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
from tetranerf.b200 import synthetic as syn  # noqa: E402


def _timed(fn, n, warm):
    ts = []
    for i in range(warm + n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        if i >= warm:
            ts.append(e0.elapsed_time(e1))
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, nargs="+", default=[45000, 300000])
    ap.add_argument("--threshold", type=float, default=0.01)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("occupancy_bench needs a GPU")
    from tetranerf import cpp
    from tetranerf.b200.render import FusedRenderer, RenderSettings

    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    st = RenderSettings.tetra_nerf()
    for n in a.points:
        V, C = syn.delaunay_mesh(n, seed=0)
        field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
        tr = cpp.TetrahedraTracer(dev)
        xyz, cells = torch.from_numpy(V).to(dev), torch.from_numpy(C).to(dev)
        tr.load_tetrahedra(xyz, cells)
        fr = FusedRenderer(tr)
        fr.set_field(torch.from_numpy(field).to(dev))
        fr.set_weights(params)
        occ = torch.zeros(len(C), dtype=torch.float32, device=dev)
        t_upd = _timed(lambda: fr.update_occupancy(occ, 0.0), a.iters, a.warmup)
        res = {"case": "occupancy", "points": n, "tetrahedra": len(C), "threshold": a.threshold,
               "update_ms": round(float(np.median(t_upd)), 3)}
        o4, d4 = (torch.from_numpy(x).to(dev) for x in syn.camera_rays(4096, seed=5000))
        o8, d8 = (torch.from_numpy(x).to(dev) for x in syn.camera_rays(8192, seed=5001))
        g = torch.Generator(device="cpu").manual_seed(1)
        jc = torch.rand((8192, st.num_samples + 1), generator=g).to(dev)
        jf = torch.rand((8192, st.num_fine_samples + 1), generator=g).to(dev)
        g_rgb = (torch.randn((8192, 3), generator=g) * 1e-3).to(dev)
        S2 = st.num_samples + st.num_fine_samples + 1
        for prec, name in ((2, "f16w2"), (3, "bf16x3")):
            fr.set_mlp_precision(prec)
            times = {False: [], True: []}
            for i in range(a.warmup + a.iters):
                for cull in (False, True):
                    fr.set_occupancy(occ if cull else None, a.threshold)
                    t = _timed(lambda: fr.render(o4, d4, st), 1, 0)[0]
                    if i >= a.warmup:
                        times[cull].append(t)
            res[f"render_ms_{name}"] = round(float(np.median(times[False])), 3)
            res[f"render_ms_{name}_culled"] = round(float(np.median(times[True])), 3)
        # culled fractions of the last culled render
        bufs = fr.debug_buffers()
        fr.set_occupancy(occ, a.threshold)
        fr.render(o4, d4, st)
        torch.cuda.synchronize()
        import ctypes

        cudart = ctypes.CDLL("libcudart.so")

        def grab(ptr, shape):
            t = torch.empty(shape, dtype=torch.int32, device=dev)
            cudart.cudaMemcpy(ctypes.c_void_p(t.data_ptr()), ctypes.c_void_p(ptr), ctypes.c_size_t(t.numel() * 4), ctypes.c_int(3))
            return t

        na = int(grab(bufs["n_active"], (1,))[0])
        for key, S, nm in (("vi_c", st.num_samples, "coarse"), ("vi_f", S2, "fine")):
            v = grab(bufs[key], (na, S, 4))
            res[f"culled_{nm}"] = round(((v[..., 0] == -1) & (v[..., 3] == -2)).float().mean().item(), 4)
        times = {False: [], True: []}
        for i in range(a.warmup + a.iters):
            for cull in (False, True):
                fr.set_occupancy(occ if cull else None, a.threshold)

                def step():
                    _, state = fr.train_forward_saved(o8, d8, st, jc, jf)
                    fr.train_backward_saved(state, g_rgb, None, len(V))

                t = _timed(step, 1, 0)[0]
                if i >= a.warmup:
                    times[cull].append(t)
        res["train_ms"] = round(float(np.median(times[False])), 3)
        res["train_ms_culled"] = round(float(np.median(times[True])), 3)
        fr.set_occupancy(None)
        res["gpu"] = gpu
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
