"""Cost and effect of Delaunay flips (DESIGN §4.19).  Needs a GPU.  Every JSON line carries the card and its power limit, read in the same
run.  On Delaunay meshes of 45k and 300k points (~0.30 M and ~2.02 M tetrahedra) after three refinement passes of 5 % random candidates:
  (a) certified-illegal interior faces before and after, the passes to the fixed point and the faces left stuck there;
  (b) the median time (CUDA events) of the first pass on the refined mesh, through the C entry point on preallocated buffers and through
      the Python call (which also allocates the workspace and outputs), its workspace, the time of every pass to the fixed point through
      the Python call, and the tracer reload;
  (c) for 4096 camera rays before and after: the mean num_visited_cells, the rays that needed the exact stage (tn_debug_trace_stats
      out2[1]), and the median time of a fused eval render (tetra-nerf settings) under synthetic.surface_scene."""
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


def _refined(xyz, cells, passes=3, frac=0.05, seed=0):
    from tetranerf.b200 import refine as rf

    g = torch.Generator(device=DEV).manual_seed(seed)
    for _ in range(passes):
        cand = torch.rand(len(cells), generator=g, device=DEV) < frac
        out = rf.refine_edges(xyz, cells, cand)
        xyz, cells = rf.migrate_vertices(xyz, out["parent_edge"], 0), out["cells"]
    return xyz.contiguous(), cells.contiguous()


def _rays_and_render(xyz, cells, field, params, o, d):
    from tetranerf import cpp
    from tetranerf.b200.render import FusedRenderer, RenderSettings

    tr = cpp.TetrahedraTracer(DEV)
    tr.load_tetrahedra(xyz, cells)
    recs = float(tr.trace_rays(o, d, 1024)["num_visited_cells"].float().mean())
    walk, exact = tr.trace_stats()
    fr = FusedRenderer(tr)
    fr.set_field(field)
    fr.set_weights(params)
    st = RenderSettings.tetra_nerf()
    t_render = _timed(lambda: fr.render(o, d, st), 10, 3)
    return {"walk": walk, "records_per_ray": round(recs, 2), "exact_stage_rays": exact, "eval_render_ms": round(t_render, 3)}


def event(points, gpu):
    from tetranerf import cpp
    from tetranerf.b200 import flip as fl

    V, Cc = syn.delaunay_mesh(points, seed=0)
    xyz, cells = _refined(torch.from_numpy(V).to(DEV), torch.from_numpy(Cc).to(DEV))
    field, params = syn.surface_scene(xyz.cpu().numpy(), 100, orc.init_mlp_params(0))
    field = torch.from_numpy(field).to(DEV)
    T = len(cells)
    nbytes = C.c_size_t(0)
    cpp._lib.tn_flip_delaunay(0, xyz.data_ptr(), len(xyz), cells.data_ptr(), T, 0xFFFFFFFF, None, None, None, None, C.byref(nbytes), None)
    # one pass through the C entry point on preallocated buffers (its kernels, sorts, scans and two small read-backs), and through the
    # Python call, which also allocates the workspace and the outputs
    ws = torch.empty((nbytes.value,), dtype=torch.uint8, device=DEV)
    c_out = torch.empty((T + T // 2, 4), dtype=torch.int32, device=DEV)
    c_src = torch.empty((T + T // 2, 3), dtype=torch.int32, device=DEV)
    counts = (C.c_uint32 * 4)()
    stream = torch.cuda.current_stream(DEV).cuda_stream
    args = (0, xyz.data_ptr(), len(xyz), cells.data_ptr(), T, 0xFFFFFFFF, c_out.data_ptr(), c_src.data_ptr(), counts, ws.data_ptr(),
            C.byref(nbytes), stream)
    assert cpp._lib.tn_flip_delaunay(*args) == 0
    t_call = _timed(lambda: cpp._lib.tn_flip_delaunay(*args), 10, 2)
    t_pass = _timed(lambda: fl.flip_delaunay(xyz, cells), 10, 2)
    passes, c1 = [], cells
    for _ in range(200):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fl.flip_delaunay(xyz, c1)
        e1.record()
        e1.synchronize()
        passes.append({"illegal": out["n_illegal"], "proposed": out["n_proposed"], "flips_23": out["n_23"], "flips_32": out["n_32"],
                       "ms": round(e0.elapsed_time(e1), 3)})
        if out["n_proposed"] == 0:
            break
        c1 = out["cells"]
    tr1 = cpp.TetrahedraTracer(DEV)
    t_reload = _timed(lambda: tr1.load_tetrahedra(xyz, c1), 5, 1)
    o, d = syn.camera_rays(4096, seed=5)
    o, d = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    before = _rays_and_render(xyz, cells, field, params, o, d)
    after = _rays_and_render(xyz, c1, field, params, o, d)
    print(json.dumps({"bench": "flip_delaunay", "gpu": gpu, "points": points, "vertices": len(xyz), "tetrahedra_before": T,
                      "tetrahedra_after": len(c1), "illegal_before": passes[0]["illegal"], "illegal_stuck": passes[-1]["illegal"],
                      "passes_to_fixed_point": len(passes) - 1, "first_pass_call_ms": round(t_call, 3),
                      "first_pass_python_ms": round(t_pass, 3), "all_passes_ms": round(sum(p["ms"] for p in passes), 2),
                      "workspace_MB": round(nbytes.value / 1e6, 1), "tracer_reload_ms": round(t_reload, 2), "before": before,
                      "after": after, "passes": passes}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, nargs="*", default=[45_000, 300_000])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("flip_bench needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    for n in a.points:
        event(n, gpu)


if __name__ == "__main__":
    main()
