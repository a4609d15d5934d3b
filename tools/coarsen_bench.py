"""Cost and effect of mesh coarsening (DESIGN §4.18).  Needs a GPU.  Every JSON line carries the card and its power limit, read in the
same run.  On Delaunay meshes of 45k and 300k points (~0.30 M and ~2.02 M tetrahedra) under synthetic.surface_scene, with its occupancy
(decay 0) and threshold 0.01, coarsen_passes = 3:
  (a) the median time of one tn_coarsen_vertices pass (CUDA events), its workspace, the tracer reload, and the whole
      TetrahedraNerf.coarsen with RAdam state to migrate; proposals and removals per pass;
  (b) vertices, tetrahedra and the mean num_visited_cells of 4096 camera rays before and after;
  (c) the median time of a 4096-ray trace, a 4096-ray fused eval render (tetra-nerf settings, culling on) and an 8192-ray fused training
      step (forward + backward + RAdam step) before and after, and the largest difference of the eval render (uniform sampler)."""
from __future__ import annotations

import argparse
import ctypes as C
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

DEV = torch.device("cuda:0")


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
    return float(np.median(ts))


def _model(V, Cc, field, params, **cfg):
    from tetranerf.nerfstudio import model as M

    config = M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(Cc), **cfg)
    m = M.TetrahedraNerf(config)
    sd = {"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(Cc), "tetrahedra_field": torch.from_numpy(field),
          "tetrahedra_occupancy": torch.zeros(len(Cc))}
    sd.update(params)
    m.load_state_dict(sd, strict=False)
    return m.to(DEV), M


def _measure(m, M, bundle, image, eval_bundle, opt):
    """trace / eval render / training step times and mean records per ray on the model's current mesh"""
    tr = m.get_tetrahedra_tracer()
    o, d = eval_bundle.origins, eval_bundle.directions
    recs = float(tr.trace_rays(o, d, 1024)["num_visited_cells"].float().mean())
    t_trace = _timed(lambda: tr.trace_rays(o, d, 512), 10, 2)
    m.eval()
    with torch.no_grad():
        t_render = _timed(lambda: m(eval_bundle), 10, 2)
    m.train()

    def step():
        opt.zero_grad(set_to_none=True)
        sum(m.get_loss_dict(m(bundle), {"image": image}).values()).backward()
        opt.step()

    t_step = _timed(step, 10, 3)
    return {"vertices": len(m.tetrahedra_vertices), "tetrahedra": len(m.tetrahedra_cells), "records_per_ray": round(recs, 2),
            "trace_ms": round(t_trace, 3), "eval_render_ms": round(t_render, 3), "train_step_ms": round(t_step, 3)}


def _render_diff(V, Cc, field, params, occ, out):
    """largest |before - after| of rgb / accumulation / expected depth of a 4096-ray fused eval render (uniform sampler, culling on)"""
    from tetranerf import cpp
    from tetranerf.b200.render import FusedRenderer, RenderSettings

    o, d = syn.camera_rays(4096, seed=4)
    o, d = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    st = RenderSettings(max_intersected_triangles=1024, num_samples=128, num_fine_samples=128, use_biased_sampler=False)
    res = []
    for x, c, f, oc in out:
        tr = cpp.TetrahedraTracer(DEV)
        tr.load_tetrahedra(x, c)
        fr = FusedRenderer(tr)
        fr.set_field(f.contiguous())
        fr.set_weights(params)
        fr.set_occupancy(oc, 0.01)
        res.append({k: v.clone() for k, v in fr.render(o, d, st, expected_depth=True).items()})
    return {k: float((res[0][k] - res[1][k]).abs().max()) for k in ("rgb", "accumulation", "expected_depth")}


def event(points, gpu):
    from tetranerf import cpp
    from tetranerf.b200 import coarsen as cv
    from tetranerf.b200.refine import migrate_cells
    from tetranerf.b200.render import FusedRenderer

    V, Cc = syn.delaunay_mesh(points, seed=0)
    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    xyz, cells, f = torch.from_numpy(V).to(DEV), torch.from_numpy(Cc).to(DEV), torch.from_numpy(field).to(DEV)
    T = len(Cc)
    tr = cpp.TetrahedraTracer(DEV)
    tr.load_tetrahedra(xyz, cells)
    fr = FusedRenderer(tr)
    fr.set_field(f)
    fr.set_weights(params)
    occ = fr.update_occupancy(torch.zeros(T, device=DEV), 0.0).clone()
    empty = occ < 0.01
    nbytes = C.c_size_t(0)
    cpp._lib.tn_coarsen_vertices(0, xyz.data_ptr(), len(V), cells.data_ptr(), T, empty.data_ptr(), 0, None, None, None, None, None,
                                 C.byref(nbytes), None)
    t_pass = _timed(lambda: cv.coarsen_vertices(xyz, cells, empty), 10, 2)
    # the passes the model makes, replayed on the bare mesh for the render comparison and the tracer reload
    x1, c1, f1, o1 = xyz, cells, f, occ
    for _ in range(3):
        out = cv.coarsen_vertices(x1, c1, o1 < 0.01)
        x1, f1 = cv.compact_vertices(x1, out["kept_vertex"], 0), cv.compact_vertices(f1, out["kept_vertex"], 1)
        c1, o1 = out["cells"], migrate_cells(o1, out["parent_cell"])
    tr1 = cpp.TetrahedraTracer(DEV)
    t_reload = _timed(lambda: tr1.load_tetrahedra(x1, c1), 5, 1)
    diff = _render_diff(V, Cc, field, params, occ, [(xyz, cells, f, occ), (x1, c1, f1, o1)])
    # the model: tetra-nerf settings (biased sampler), culling on, RAdam state from real steps
    m, M = _model(V, Cc, field, params, num_samples=128, num_fine_samples=128, use_biased_sampler=True, use_occupancy_field=True,
                  occupancy_warmup_steps=0, occupancy_update_interval=10**9, coarsen_every=1, coarsen_passes=3,
                  max_intersected_triangles=1024)
    opt = torch.optim.RAdam(list(m.parameters()), lr=1e-4)
    o, d = syn.camera_rays(8192, seed=3)
    bundle = M.RayBundle(origins=torch.from_numpy(o).to(DEV), directions=torch.from_numpy(d).to(DEV))
    eo, ed = syn.camera_rays(4096, seed=5)
    eval_bundle = M.RayBundle(origins=torch.from_numpy(eo).to(DEV), directions=torch.from_numpy(ed).to(DEV))
    image = torch.rand((8192, 3), generator=torch.Generator().manual_seed(1)).to(DEV)
    before = _measure(m, M, bundle, image, eval_bundle, opt)
    res = m.coarsen(opt)
    after = _measure(m, M, bundle, image, eval_bundle, opt)
    print(json.dumps({"bench": "coarsen_event", "gpu": gpu, "tetrahedra": T, "vertices": len(V), "empty_fraction": round(float(empty.float().mean()), 4),
                      "coarsen_vertices_ms": round(t_pass, 3), "workspace_MB": round(nbytes.value / 1e6, 1),
                      "tracer_reload_ms": round(t_reload, 2), "coarsen_ms": round(res["seconds"] * 1e3, 2), "passes": res["passes"],
                      "before": before, "after": after, "max_render_diff": diff}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, nargs="*", default=[45_000, 300_000])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("coarsen_bench needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    for n in a.points:
        event(n, gpu)


if __name__ == "__main__":
    main()
