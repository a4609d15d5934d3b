"""Cost and gain of mesh refinement (DESIGN §4.14).  Needs a GPU.  Every JSON line carries the card and its power limit, read in the
same run.
  (a) one refinement event on Delaunay meshes of 45k and 300k points (~0.30 M and ~2.02 M tetrahedra), 5 % candidates (random
      scores), refine_passes = 3: the median time of one tn_refine_edges pass (CUDA events), its workspace, the tracer reload, and the
      whole TetrahedraNerf.refine with RAdam state to migrate; the acceptances per pass;
  (b) the median time of an 8192-ray fused training step (forward + backward + RAdam step, CUDA events) before and after that event;
  (c) quality: surface_scene with noise 0, the MLP held fixed, the field alone trained with RAdam toward the eval renders of the
      45k-point mesh, from a 4k-point mesh; arms over the same steps: the 4k mesh as is, the same mesh with refinement, and a fresh
      Delaunay mesh with as many vertices as the refined one ends with.  PSNR against held-out rays."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import time
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
    sd = {"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(Cc), "tetrahedra_field": torch.from_numpy(field)}
    sd.update(params)
    m.load_state_dict(sd, strict=False)
    return m.to(DEV), M


def _train_step(m, M, opt, bundle, image):
    opt.zero_grad(set_to_none=True)
    loss = sum(m.get_loss_dict(m(bundle), {"image": image}).values())
    loss.backward()
    opt.step()


def event_cost(points, gpu):
    from tetranerf import cpp
    from tetranerf.b200 import refine as rf

    V, Cc = syn.delaunay_mesh(points, seed=0)
    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    xyz, cells = torch.from_numpy(V).to(DEV), torch.from_numpy(Cc).to(DEV)
    T = len(Cc)
    g = torch.Generator(device=DEV).manual_seed(0)
    cand = torch.rand(T, generator=g, device=DEV) < 0.05
    nbytes = C.c_size_t(0)
    cpp._lib.tn_refine_edges(0, xyz.data_ptr(), len(V), cells.data_ptr(), T, cand.data_ptr(), 0.0, 0, None, None, None, None, None,
                             C.byref(nbytes), None)
    t_pass = _timed(lambda: rf.refine_edges(xyz, cells, cand), 10, 2)
    out = rf.refine_edges(xyz, cells, cand)
    x1 = rf.migrate_vertices(xyz, out["parent_edge"], 0)
    tr = cpp.TetrahedraTracer(DEV)
    tr.load_tetrahedra(x1, out["cells"])
    t_reload = _timed(lambda: tr.load_tetrahedra(x1, out["cells"]), 5, 1)
    # the whole refine() inside a training loop: statistics from real steps, then random scores so 5 % of the tetrahedra are candidates
    m, M = _model(V, Cc, field, params, refine_every=1, refine_fraction=0.05, refine_passes=3, num_samples=128, num_fine_samples=128,
                  use_biased_sampler=True)
    opt = torch.optim.RAdam(list(m.parameters()), lr=1e-3)
    o, d = syn.camera_rays(8192, seed=3)
    bundle = M.RayBundle(origins=torch.from_numpy(o).to(DEV), directions=torch.from_numpy(d).to(DEV))
    image = torch.rand((8192, 3), generator=torch.Generator().manual_seed(1)).to(DEV)
    m.train()
    step = lambda: _train_step(m, M, opt, bundle, image)  # noqa: E731
    t_step0 = _timed(step, 10, 3)
    m._grad_acc = torch.rand(len(V), generator=g, device=DEV)
    m._grad_cnt = torch.ones(len(V), dtype=torch.int32, device=DEV)
    res = m.refine(opt)
    t_step1 = _timed(step, 10, 3)
    print(json.dumps({"bench": "refine_event", "gpu": gpu, "tetrahedra": T, "vertices": len(V), "candidates": int(cand.sum()),
                      "refine_edges_ms": round(t_pass, 3), "workspace_MB": round(nbytes.value / 1e6, 1),
                      "accepted_one_pass": out["n_accepted"], "split_one_pass": out["n_split"], "tracer_reload_ms": round(t_reload, 2),
                      "refine_ms": round(res["seconds"] * 1e3, 2), "passes": res["passes"], "tetrahedra_after": res["tetrahedra_after"],
                      "vertices_after": res["vertices_after"], "train_step_ms_before": round(t_step0, 3),
                      "train_step_ms_after": round(t_step1, 3)}), flush=True)


def quality(gpu, steps, base_points, every):
    from tetranerf.b200.render import FusedRenderer, RenderSettings
    from tetranerf import cpp

    params0 = orc.init_mlp_params(0)
    Vt, Ct = syn.delaunay_mesh(45_000, seed=0)
    ft, params = syn.surface_scene(Vt, 100, params0, noise=0.0)
    st = RenderSettings(num_samples=64, num_fine_samples=64)
    tr = cpp.TetrahedraTracer(DEV)
    tr.load_tetrahedra(torch.from_numpy(Vt).to(DEV), torch.from_numpy(Ct).to(DEV))
    fr = FusedRenderer(tr)
    fr.set_field(torch.from_numpy(ft).to(DEV))
    fr.set_weights(params)
    fr.set_mlp_precision(3)

    def rays(n, seed):
        o, d = syn.camera_rays(n, seed=seed)
        o, d = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
        return o, d, fr.render(o, d, st)["rgb"].clone()

    train = [rays(8192, 100 + i) for i in range(8)]
    held = rays(16384, 7)

    def arm(V, Cc, refine):
        f, _ = syn.surface_scene(V, 100, params0, noise=0.0)
        m, M = _model(V, Cc, f, params, num_samples=64, num_fine_samples=64, refine_every=every if refine else 0, refine_start=every,
                      refine_stop=steps - every, refine_fraction=0.05, refine_passes=3)
        for n, p in m.named_parameters():
            p.requires_grad_(n == "tetrahedra_field")
        opt = torch.optim.RAdam([m.tetrahedra_field], lr=1e-2)
        cbs = m.get_training_callbacks(M.TrainingCallbackAttributes(optimizers={"fields": opt}))
        m.train()
        for s in range(1, steps + 1):
            o, d, img = train[s % len(train)]
            _train_step(m, M, opt, M.RayBundle(origins=o, directions=d), img)
            for cb in cbs:
                cb.run_callback_at_location(s, M.TrainingCallbackLocation.AFTER_TRAIN_ITERATION)
        m.eval()
        with torch.no_grad():
            got = m(M.RayBundle(origins=held[0], directions=held[1]))["rgb"]
        psnr = float(10 * torch.log10(1.0 / torch.mean((got - held[2]) ** 2)))
        return psnr, len(m.tetrahedra_vertices), len(m.tetrahedra_cells)

    V, Cc = syn.delaunay_mesh(base_points, seed=1)
    t0 = time.perf_counter()
    p_base = arm(V, Cc, False)
    p_ref = arm(V, Cc, True)
    Vf, Cf = syn.delaunay_mesh(p_ref[1], seed=1)
    p_uni = arm(Vf, Cf, False)
    print(json.dumps({"bench": "refine_quality", "gpu": gpu, "steps": steps, "refine_every": every,
                      "base": {"psnr": round(p_base[0], 3), "vertices": p_base[1], "tetrahedra": p_base[2]},
                      "refined": {"psnr": round(p_ref[0], 3), "vertices": p_ref[1], "tetrahedra": p_ref[2]},
                      "uniform_same_vertices": {"psnr": round(p_uni[0], 3), "vertices": p_uni[1], "tetrahedra": p_uni[2]},
                      "seconds": round(time.perf_counter() - t0, 1)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, nargs="*", default=[45_000, 300_000])
    ap.add_argument("--quality-steps", type=int, default=1500)
    ap.add_argument("--quality-every", type=int, default=250)
    ap.add_argument("--base-points", type=int, default=4000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("refine_bench needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    for n in a.points:
        event_cost(n, gpu)
    if a.quality_steps > 0:
        quality(gpu, a.quality_steps, a.base_points, a.quality_every)


if __name__ == "__main__":
    main()
