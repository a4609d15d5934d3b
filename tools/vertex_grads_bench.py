"""Cost of the vertex gradient and of the in-place refit (DESIGN §4.9), on bench.py --mode train's workload (8192 rays, the 300k-point /
2.02 M-tetrahedra mesh, the tetra_nerf configuration, a random field and the torch-default network).  Prints JSON lines:
  * per mode (default / deterministic): median training step (saved forward + backward) without and with the vertex gradient, alternating,
    and the extra device memory of the backward with it;
  * update_vertices against load_tetrahedra on that mesh (median of alternating runs);
  * trace_rays after a refit to a perturbation of 0.1 x the median edge length against a fresh load at the same positions (the cost of
    keeping the load's Morton order).
with the card and its power limit.  Needs a GPU."""
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
from tetranerf import cpp  # noqa: E402
from tetranerf.b200 import synthetic as syn  # noqa: E402
from tetranerf.b200.render import FusedRenderer, RenderSettings  # noqa: E402


def _time(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=8192)
    ap.add_argument("--points", type=int, default=300_000)
    ap.add_argument("--iters", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vertex_grads_bench needs a GPU")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    V, C = syn.delaunay_mesh(a.points, seed=0)
    xyz, cells = torch.from_numpy(V).to(dev), torch.from_numpy(C).to(dev)
    tr = cpp.TetrahedraTracer(dev)
    tr.load_tetrahedra(xyz, cells)
    fr = FusedRenderer(tr)
    fr.set_field(torch.from_numpy(syn.random_field(len(V), 64, seed=3, kind="init")).to(dev))
    fr.set_weights(orc.init_mlp_params(0))
    st = RenderSettings.tetra_nerf()
    o, d = (torch.from_numpy(x).to(dev) for x in syn.camera_rays(a.rays, seed=5000))
    g = torch.Generator().manual_seed(9)
    jc, jf = torch.rand((a.rays, st.num_samples + 1), generator=g).to(dev), torch.rand((a.rays, st.num_fine_samples + 1), generator=g).to(dev)
    target = torch.rand((a.rays, 3), generator=g).to(dev)

    def step(gv: bool):
        out, state = fr.train_forward_saved(o, d, st, jc, jf)
        g_rgb = (2.0 * (out["rgb"] - target) / (3 * a.rays)).contiguous()
        fr.train_backward_saved(state, g_rgb, None, len(V), True, grad_vertices=gv)

    for det in (False, True):
        os.environ["TETRANERF_B200_DETERMINISTIC"] = "1" if det else "0"
        step(False)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info(dev)[0]
        step(True)
        torch.cuda.synchronize()
        extra = free0 - torch.cuda.mem_get_info(dev)[0]
        times = {False: [], True: []}
        for it in range(a.warmup + a.iters):
            for gv in (False, True):
                t = _time(lambda: step(gv))
                if it >= a.warmup:
                    times[gv].append(t)
        plain, with_v = float(np.median(times[False])), float(np.median(times[True]))
        print(json.dumps({"what": "train_step", "mode": "deterministic" if det else "default", "rays": a.rays, "tetrahedra": len(C),
                          "iters": a.iters, "step_ms": round(plain, 3), "step_ms_with_vertex_grads": round(with_v, 3),
                          "extra_ms": round(with_v - plain, 3), "extra_device_bytes": int(extra), "gpu": q}), flush=True)

    # refit against a fresh load of the same mesh
    edge = float(np.median(np.linalg.norm(V[C[:, 1]] - V[C[:, 0]], axis=-1)))
    P = torch.from_numpy((V + 0.1 * edge * np.random.default_rng(1).standard_normal(V.shape)).astype(np.float32)).to(dev)
    other = cpp.TetrahedraTracer(dev)
    other.load_tetrahedra(P, cells)
    t_up, t_load = [], []
    for it in range(a.warmup + a.iters):
        u = _time(lambda: tr.update_vertices(P if it % 2 == 0 else xyz))
        ld = _time(lambda: other.load_tetrahedra(P, cells))
        if it >= a.warmup:
            t_up.append(u)
            t_load.append(ld)
    folded, walkable = tr.update_vertices(P)
    print(json.dumps({"what": "refit", "tetrahedra": len(C), "update_vertices_ms": round(float(np.median(t_up)), 3),
                      "load_tetrahedra_ms": round(float(np.median(t_load)), 3), "folded_faces_at_0.1_edge": folded, "walkable": walkable,
                      "gpu": q}), flush=True)
    # trace after the refit (the load's Morton order, grown boxes) against the fresh load at the same positions
    for impl, walk in (("default", None), ("bvh", (2**32 - 1, (1, 0), (1, 0)))):  # the batch-size default first, then forced
        for t in (tr, other):
            if walk is not None:
                t.set_walk_min_rays(walk[0]); t.set_walk_solo_range(*walk[1]); t.set_walk_quad_range(*walk[2])
        ta, tb = [], []
        for it in range(a.warmup + a.iters):
            x = _time(lambda: tr.trace_rays(o, d, st.max_intersected_triangles))
            y = _time(lambda: other.trace_rays(o, d, st.max_intersected_triangles))
            if it >= a.warmup:
                ta.append(x)
                tb.append(y)
        tr.synchronize()
        print(json.dumps({"what": "trace_after_refit", "impl": impl, "rays": a.rays, "refit_ms": round(float(np.median(ta)), 3),
                          "fresh_load_ms": round(float(np.median(tb)), 3), "gpu": q}), flush=True)


if __name__ == "__main__":
    main()
